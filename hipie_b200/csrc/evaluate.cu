// Evaluation reductions on the device (reference: detectron2/evaluation/sem_seg_evaluation.py SemSegEvaluator.process and
// panopticapi's pq_compute_single_core, driven by COCOPanopticEvaluator).  The reference copies every argmax map to the host and
// runs np.bincount on it, and encodes / decodes a PNG per image to run np.unique on the id maps; here both reductions run next to
// the model's outputs and only the counters leave the device.
//   semseg_confusion  one pass over the (C, H, W) class scores: the first-index argmax over C per pixel (torch.argmax), the GT label
//                     (ignore -> C), and conf[pred, gt] += 1 into the (C + 1)^2 int64 matrix.  The argmax map is never stored.
//   panoptic_pairs    one pass over the predicted segment ids and the RGB-coded GT PNG: table[gt row, pred id] += 1 with the GT id
//                     R + 256 G + 65536 B decoded in the kernel and looked up in the image's listed segment ids.
// Both kernels aggregate equal keys within a warp (__match_any_sync) before one global atomic per distinct key: most pixels of a warp
// fall in one or two (pred, gt) pairs, so the matrix sees a few atomics per 32 pixels instead of 32.
#include <algorithm>

#include "common.cuh"

namespace hipie {

constexpr int EV_THREADS = 256;
constexpr int EV_UNROLL = 16;          // class planes in flight per thread: the loads of one group are independent
constexpr int EV_MAX_CLASSES = 4096;  // a (C + 1)^2 int64 matrix of at most 134 MB
constexpr int PP_MAX_GT = 4096;        // listed GT segments per image (shared-memory lookup table)
constexpr int PP_MAX_PRED = 65535;     // predicted segment ids 1..S
constexpr int64_t PP_MAX_TABLE = 1ll << 24;      // table entries (128 MB of int64)

// Adds 1 per lane to hist[key] for every lane with key >= 0, one atomic per distinct key of the warp.  Every lane of the warp calls it.
__device__ __forceinline__ void warp_count(int64_t key, unsigned long long* hist) {
    const unsigned same = __match_any_sync(0xffffffffu, key);
    const int lane = threadIdx.x & 31;
    if (key >= 0 && lane == __ffs(same) - 1) atomicAdd(hist + key, (unsigned long long)__popc(same));
}

// Grid-stride over pixels, one pixel per thread per step, every lane of a warp on the same step (out-of-range lanes carry key -1), so
// the C plane loads of a warp are 128 consecutive bytes of each plane.
__global__ void __launch_bounds__(EV_THREADS)
semseg_confusion_kernel(const float* __restrict__ sem, int C, int64_t HW, const int* __restrict__ gt, int ignore_label,
                        unsigned long long* __restrict__ conf, unsigned long long* __restrict__ err) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p - threadIdx.x % 32 < HW; p += stride) {
        int64_t key = -1;
        if (p < HW) {
            const float* s = sem + p;
            float best = __ldg(s);
            int arg = 0;
            int c0 = 1;
            for (; c0 + EV_UNROLL <= C; c0 += EV_UNROLL) {
                float v[EV_UNROLL];
#pragma unroll
                for (int u = 0; u < EV_UNROLL; ++u) v[u] = __ldg(s + (int64_t)(c0 + u) * HW);
#pragma unroll
                for (int u = 0; u < EV_UNROLL; ++u)
                    if (beats(v[u], best)) { best = v[u]; arg = c0 + u; }
            }
            for (; c0 < C; ++c0) {
                const float v = __ldg(s + (int64_t)c0 * HW);
                if (beats(v, best)) { best = v; arg = c0; }
            }
            int g = __ldg(gt + p);
            if (g == ignore_label) g = C;
            else if (g < 0 || g >= C) g = -1;                   // a label the matrix has no column for: counted, not binned
            if (g < 0) atomicAdd(err, 1ull);
            else key = (int64_t)arg * (C + 1) + g;
        }
        warp_count(key, conf);
    }
}

__global__ void __launch_bounds__(EV_THREADS)
panoptic_pairs_kernel(const int* __restrict__ pred, const uint8_t* __restrict__ gt_rgb, int64_t HW, const int* __restrict__ gt_ids, int n_gt,
                      int S, unsigned long long* __restrict__ table, unsigned long long* __restrict__ err) {
    __shared__ int ids[PP_MAX_GT];
    for (int i = threadIdx.x; i < n_gt; i += blockDim.x) ids[i] = gt_ids[i];
    __syncthreads();
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p - threadIdx.x % 32 < HW; p += stride) {
        int64_t key = -1;
        if (p < HW) {
            const uint8_t* c = gt_rgb + 3 * p;
            const int id = (int)c[0] + 256 * (int)c[1] + 65536 * (int)c[2];
            int row = 0;                                        // GT id 0 is VOID
            if (id != 0) {
                int lo = 0, hi = n_gt;                          // first listed id >= id
                while (lo < hi) {
                    const int mid = (lo + hi) >> 1;
                    if (ids[mid] < id) lo = mid + 1;
                    else hi = mid;
                }
                row = (lo < n_gt && ids[lo] == id) ? lo + 1 : n_gt + 1;      // n_gt + 1: present in the PNG, not listed
            }
            const int q = __ldg(pred + p);
            if (q < 0 || q > S) atomicAdd(err, 1ull);
            else key = (int64_t)row * (S + 1) + q;
        }
        warp_count(key, table);
    }
}

static int ev_grid(int64_t HW) { return (int)std::max<int64_t>(1, std::min<int64_t>((HW + EV_THREADS - 1) / EV_THREADS, (int64_t)num_sms() * 8)); }

// ---- instance overlaps (pycocotools maskApi.c rleIou, as COCOeval.computeIoU runs it on the RLEs of COCOEvaluator.process).  One bit
// layout for predictions and GTs: a mask is its flattened row-major pixels (bit j of word w = pixel y * W + x = 32 w + j), K = H * W
// zero-padded to whole 256-bit chunks, so one mask row is KW = ceil(K / 256) * 8 words and both operands of the overlap MMA are
// K-contiguous.
constexpr int IO_MAX_PRED = 1024;
constexpr int IO_MAX_GT = 4096;
constexpr int PK_THREADS = 256;
constexpr int PK_UNROLL = 16;            // words (independent 32-byte loads) per warp and step
constexpr int OV_THREADS = 128;          // 2 x 2 warps, each a 32 x 32 tile of (prediction, GT) pairs
constexpr int OV_TILE = 64;

static int64_t mask_words(int64_t HW) { return (HW + 255) / 256 * 8; }

// Pack: each warp turns 32 consecutive bytes into one word with a ballot; PK_UNROLL such loads are in flight per lane, so a warp reads a
// contiguous 512-byte span per step.  Words past ceil(K / 32) come out zero.  area[n] = the mask's pixel count.
__global__ void __launch_bounds__(PK_THREADS)
mask_pack_kernel(const uint8_t* __restrict__ masks, int64_t HW, int64_t KW, uint32_t* __restrict__ bits, int* __restrict__ area) {
    const int n = blockIdx.y;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint8_t* m = masks + (int64_t)n * HW;
    uint32_t* out = bits + (int64_t)n * KW;
    int count = 0;
    const int64_t step = (int64_t)gridDim.x * (PK_THREADS / 32) * PK_UNROLL;
    for (int64_t w0 = ((int64_t)blockIdx.x * (PK_THREADS / 32) + warp) * PK_UNROLL; w0 < KW; w0 += step) {
        uint8_t v[PK_UNROLL];
#pragma unroll
        for (int u = 0; u < PK_UNROLL; ++u) {
            const int64_t p = (w0 + u) * 32 + lane;
            v[u] = p < HW ? __ldg(m + p) : 0;
        }
        uint32_t mine = 0;
#pragma unroll
        for (int u = 0; u < PK_UNROLL; ++u) {
            const uint32_t word = __ballot_sync(0xffffffffu, v[u] != 0);
            if (lane == u) mine = word;
        }
        if (lane < PK_UNROLL && w0 + lane < KW) {
            out[w0 + lane] = mine;
            count += __popc(mine);
        }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) count += __shfl_xor_sync(0xffffffffu, count, o);
    __shared__ int part[PK_THREADS / 32];
    if (lane == 0) part[warp] = count;
    __syncthreads();
    if (threadIdx.x == 0) {
        int s = 0;
        for (int i = 0; i < PK_THREADS / 32; ++i) s += part[i];
        if (s) atomicAdd(area + n, s);
    }
}

// Expand: one thread per output word.  ends[off[g] .. off[g + 1]) are the cumulative ends of GT g's column-major runs (background
// first); pixel (y, x) has column-major index c = x * H + y and is foreground iff the number of ends <= c is odd.  Along a row c grows
// by H, so the search of the next pixel starts at the previous run.  A list whose last end is not H * W is counted in *err.
__global__ void __launch_bounds__(EV_THREADS)
rle_expand_kernel(const int* __restrict__ ends, const int64_t* __restrict__ off, int M, int H, int W, int64_t KW, uint32_t* __restrict__ bits,
                  unsigned long long* __restrict__ err) {
    const int64_t HW = (int64_t)H * W;
    const int64_t total = (int64_t)M * KW;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int g = (int)(i / KW);
        const int64_t w = i - (int64_t)g * KW;
        const int* e = ends + off[g];
        const int r = (int)(off[g + 1] - off[g]);
        if (w == 0 && (r == 0 || e[r - 1] != HW)) atomicAdd(err, 1ull);
        uint32_t word = 0;
        int64_t p = w * 32;
        if (p < HW) {
            int y = (int)(p / W), x = (int)(p - (int64_t)y * W);
            int lo = 0;
            for (int j = 0; j < 32 && p + j < HW; ++j) {
                const int c = x * H + y;                        // < H * W < 2^31
                int hi = r;                                     // first end > c, searched in [lo, r)
                while (lo < hi) {
                    const int mid = (lo + hi) >> 1;
                    if (__ldg(e + mid) <= c) lo = mid + 1;
                    else hi = mid;
                }
                word |= (uint32_t)(lo & 1) << j;
                if (++x == W) { x = 0; ++y; lo = 0; }
            }
        }
        bits[i] = word;
    }
}

__device__ __forceinline__ void mma_b1_and_popc(int (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k256.row.col.s32.b1.b1.s32.and.popc {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// inter[n, m] += sum_k popc(P[n, k] & G[m, k]) over this CTA's slice of the 256-bit chunks.  Fragments come straight from global memory
// as uint2: lane (g, t) takes words 2t and 2t + 1 of a chunk for the k-blocks t and t + 4 of both A and B (the same permutation of k on
// both sides, so the popcount sum is unchanged).  Rows past N / M read zeros and are not stored.
__global__ void __launch_bounds__(OV_THREADS)
mask_overlaps_kernel(const uint32_t* __restrict__ P, int N, const uint32_t* __restrict__ G, int M, int64_t KW, int chunks_per_cta,
                     int* __restrict__ inter) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int g = lane >> 2, t = lane & 3;
    const int n_base = blockIdx.y * OV_TILE + (warp >> 1) * 32;
    const int m_base = blockIdx.x * OV_TILE + (warp & 1) * 32;
    const int64_t nchunks = KW / 8;
    const int64_t c0 = (int64_t)blockIdx.z * chunks_per_cta;
    const int64_t c1 = min(nchunks, c0 + chunks_per_cta);
    const uint2 zero = make_uint2(0u, 0u);
    const uint2* arow[4];
    bool aok[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) {                              // rows g, g + 8, g + 16, g + 24 of the warp's 32 predictions
        const int n = n_base + g + 8 * r;
        aok[r] = n < N;
        arow[r] = reinterpret_cast<const uint2*>(P + (int64_t)(aok[r] ? n : 0) * KW) + t;
    }
    const uint2* brow[4];
    bool bok[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int m = m_base + 8 * j + g;
        bok[j] = m < M;
        brow[j] = reinterpret_cast<const uint2*>(G + (int64_t)(bok[j] ? m : 0) * KW) + t;
    }
    int acc[2][4][4] = {};
#pragma unroll 2
    for (int64_t c = c0; c < c1; ++c) {
        uint2 a[4], b[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) a[r] = aok[r] ? __ldg(arow[r] + c * 4) : zero;
#pragma unroll
        for (int j = 0; j < 4; ++j) b[j] = bok[j] ? __ldg(brow[j] + c * 4) : zero;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const uint32_t af[4] = {a[2 * i].x, a[2 * i + 1].x, a[2 * i].y, a[2 * i + 1].y};
#pragma unroll
            for (int j = 0; j < 4; ++j) mma_b1_and_popc(acc[i][j], af, b[j].x, b[j].y);
        }
    }
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int q = 0; q < 4; ++q) {                      // c0, c1: row g; c2, c3: row g + 8; columns 2t, 2t + 1
                const int n = n_base + 16 * i + g + 8 * (q >> 1);
                const int m = m_base + 8 * j + 2 * t + (q & 1);
                if (n < N && m < M && acc[i][j][q]) atomicAdd(inter + (int64_t)n * M + m, acc[i][j][q]);
            }
}

}  // namespace hipie

using namespace hipie;

extern "C" int hipie_semseg_confusion(const float* sem, int C, int H, int W, const int* gt, int ignore_label, unsigned long long* conf,
                                      unsigned long long* err, void* stream) {
    HIPIE_CHECK_ARG(sem && gt && conf && err, "hipie_semseg_confusion: null pointer");
    HIPIE_CHECK_ARG(C >= 1 && C <= EV_MAX_CLASSES, "hipie_semseg_confusion: %d classes (1 .. %d)", C, EV_MAX_CLASSES);
    HIPIE_CHECK_ARG(H > 0 && W > 0 && (int64_t)H * W < (1ll << 31), "hipie_semseg_confusion: bad image size %d x %d (H * W < 2^31)", H, W);
    const int64_t HW = (int64_t)H * W;
    semseg_confusion_kernel<<<ev_grid(HW), EV_THREADS, 0, (cudaStream_t)stream>>>(sem, C, HW, gt, ignore_label, conf, err);
    HIPIE_CHECK_LAUNCH();
    return HIPIE_OK;
}

extern "C" int hipie_panoptic_pairs(const int* pred, const uint8_t* gt_rgb, int H, int W, const int* gt_ids, int n_gt, int S,
                                    unsigned long long* table, unsigned long long* err, void* stream) {
    HIPIE_CHECK_ARG(pred && gt_rgb && table && err && (n_gt == 0 || gt_ids), "hipie_panoptic_pairs: null pointer");
    HIPIE_CHECK_ARG(n_gt >= 0 && n_gt <= PP_MAX_GT, "hipie_panoptic_pairs: %d listed GT segments (at most %d)", n_gt, PP_MAX_GT);
    HIPIE_CHECK_ARG(S >= 0 && S <= PP_MAX_PRED, "hipie_panoptic_pairs: %d predicted segments (at most %d)", S, PP_MAX_PRED);
    HIPIE_CHECK_ARG((int64_t)(n_gt + 2) * (S + 1) <= PP_MAX_TABLE, "hipie_panoptic_pairs: table of %d x %d entries (at most %lld)", n_gt + 2,
                    S + 1, (long long)PP_MAX_TABLE);
    HIPIE_CHECK_ARG(H > 0 && W > 0 && (int64_t)H * W < (1ll << 31), "hipie_panoptic_pairs: bad image size %d x %d (H * W < 2^31)", H, W);
    const int64_t HW = (int64_t)H * W;
    panoptic_pairs_kernel<<<ev_grid(HW), EV_THREADS, 0, (cudaStream_t)stream>>>(pred, gt_rgb, HW, gt_ids, n_gt, S, table, err);
    HIPIE_CHECK_LAUNCH();
    return HIPIE_OK;
}

extern "C" int64_t hipie_mask_words(int H, int W) { return (H > 0 && W > 0) ? mask_words((int64_t)H * W) : 0; }

extern "C" int hipie_mask_pack(const uint8_t* masks, int N, int H, int W, uint32_t* bits, int* area, void* stream) {
    HIPIE_CHECK_ARG(N >= 0 && N <= IO_MAX_PRED, "hipie_mask_pack: %d masks (at most %d)", N, IO_MAX_PRED);
    HIPIE_CHECK_ARG(H > 0 && W > 0 && (int64_t)H * W < (1ll << 31), "hipie_mask_pack: bad image size %d x %d (H * W < 2^31)", H, W);
    if (N == 0) return HIPIE_OK;
    HIPIE_CHECK_ARG(masks && bits && area, "hipie_mask_pack: null pointer");
    const int64_t HW = (int64_t)H * W, KW = mask_words(HW);
    const int64_t per_block = (PK_THREADS / 32) * PK_UNROLL;
    const int64_t want = std::max<int64_t>(1, ((int64_t)num_sms() * 8 + N - 1) / N);
    const int gx = (int)std::max<int64_t>(1, std::min<int64_t>((KW + per_block - 1) / per_block, want));
    mask_pack_kernel<<<dim3(gx, N), PK_THREADS, 0, (cudaStream_t)stream>>>(masks, HW, KW, bits, area);
    HIPIE_CHECK_LAUNCH();
    return HIPIE_OK;
}

extern "C" int hipie_rle_expand(const int* ends, const int64_t* offsets, int M, int H, int W, uint32_t* bits, unsigned long long* err,
                                void* stream) {
    HIPIE_CHECK_ARG(M >= 0 && M <= IO_MAX_GT, "hipie_rle_expand: %d GT masks (at most %d)", M, IO_MAX_GT);
    HIPIE_CHECK_ARG(H > 0 && W > 0 && (int64_t)H * W < (1ll << 31), "hipie_rle_expand: bad image size %d x %d (H * W < 2^31)", H, W);
    if (M == 0) return HIPIE_OK;
    HIPIE_CHECK_ARG(ends && offsets && bits && err, "hipie_rle_expand: null pointer");
    const int64_t KW = mask_words((int64_t)H * W);
    const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((M * KW + EV_THREADS - 1) / EV_THREADS, (int64_t)num_sms() * 16));
    rle_expand_kernel<<<grid, EV_THREADS, 0, (cudaStream_t)stream>>>(ends, offsets, M, H, W, KW, bits, err);
    HIPIE_CHECK_LAUNCH();
    return HIPIE_OK;
}

extern "C" int hipie_mask_overlaps(const uint32_t* pred_bits, int N, const uint32_t* gt_bits, int M, int H, int W, int* inter, void* stream) {
    HIPIE_CHECK_ARG(N >= 0 && N <= IO_MAX_PRED, "hipie_mask_overlaps: %d predicted masks (at most %d)", N, IO_MAX_PRED);
    HIPIE_CHECK_ARG(M >= 0 && M <= IO_MAX_GT, "hipie_mask_overlaps: %d GT masks (at most %d)", M, IO_MAX_GT);
    HIPIE_CHECK_ARG(H > 0 && W > 0 && (int64_t)H * W < (1ll << 31), "hipie_mask_overlaps: bad image size %d x %d (H * W < 2^31)", H, W);
    if (N == 0 || M == 0) return HIPIE_OK;
    HIPIE_CHECK_ARG(pred_bits && gt_bits && inter, "hipie_mask_overlaps: null pointer");
    const int64_t KW = mask_words((int64_t)H * W), nchunks = KW / 8;
    const int tiles = ((M + OV_TILE - 1) / OV_TILE) * ((N + OV_TILE - 1) / OV_TILE);
    const int64_t splits = std::max<int64_t>(1, std::min<int64_t>(nchunks, ((int64_t)num_sms() * 4 + tiles - 1) / tiles));
    const int per = (int)((nchunks + splits - 1) / splits);
    const dim3 grid((M + OV_TILE - 1) / OV_TILE, (N + OV_TILE - 1) / OV_TILE, (unsigned)((nchunks + per - 1) / per));
    mask_overlaps_kernel<<<grid, OV_THREADS, 0, (cudaStream_t)stream>>>(pred_bits, N, gt_bits, M, KW, per, inter);
    HIPIE_CHECK_LAUNCH();
    return HIPIE_OK;
}
