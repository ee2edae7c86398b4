// Device-side selection steps of HIPIE's inference post-processing (SURVEY.md §8 row a20; reference
// /root/reference/projects/HIPIE/hipie/hipie_img.py:587-657 `inference` and :1025-1052 `convert_grounding_to_od_logits`):
//
//   hipie_class_scores   token -> class pooling (mean or max over each class's token span), FG / BG class masking with
//                        -9999, prob = sqrt(sigmoid(cls) * sigmoid(iou)), per-query max / argmax over the classes
//                        (the reference loops over the classes on the host with index tensors: 847 x 3 launches for ADE-847)
//   hipie_batched_nms    class-aware greedy NMS with torchvision's coordinate-offset formulation
//                        (torchvision.ops.batched_nms -> _batched_nms_coordinate_trick -> nms: boxes + idx * (max + 1),
//                        IoU = inter / (a + b - inter) > thr), one CTA per image: in-CTA sort, pair bit matrix, serial scan
//   hipie_topk           k largest of a row (values descending, lowest index first among equals), one CTA per row:
//                        4-pass byte radix select on the order-preserving integer image of the floats + in-CTA sort of the
//                        survivors.  Used for the flat top-100 over (kept query x class) and for the two-stage proposal top-k.
//   hipie_nms_sorted     greedy single-class NMS of up to 32768 score-sorted xyxy boxes (SAM's automatic mask generator): 64 x 64
//                        IoU tiles into a global-memory bit matrix, then one sweep
//
// All three are launch-latency sized problems (<= 1e6 elements per image); the point is that the selection runs on the
// device without host round trips or library calls, inside the same stream / CUDA graph as the rest of the path.
#include "common.cuh"
#include <float.h>

namespace hipie {

namespace {

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

// logits (R, Lt) | tok (C, maxlen) int32 token indices, padded by repeating the first | cnt (C) int32 (0 = class absent)
// mode_mask (C) int8: 1 = class is masked to -9999 (FG mode: stuff classes; BG mode: thing classes)
__global__ void class_scores_kernel(const float* __restrict__ logits, const int* __restrict__ tok, const int* __restrict__ cnt,
                                    const int8_t* __restrict__ masked, const float* __restrict__ iou, float* __restrict__ scores,
                                    float* __restrict__ prob, float* __restrict__ row_max, int* __restrict__ row_arg, int R, int Lt,
                                    int C, int maxlen, int max_pool) {
    const int r = blockIdx.x;
    if (r >= R) return;
    const float* lr = logits + (size_t)r * Lt;
    const float iou_s = iou ? sigmoidf_(iou[r]) : 1.f;
    float best = -FLT_MAX;
    int barg = 0x7fffffff;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        const int n = cnt[c];
        float s = 0.f;
        if (n > 0) {
            const int* tc = tok + (size_t)c * maxlen;
            if (max_pool) {
                s = lr[tc[0]];
                for (int j = 1; j < n; ++j) s = fmaxf(s, lr[tc[j]]);
            } else {
                for (int j = 0; j < n; ++j) s += lr[tc[j]];
                s = s / (float)n;                      // torch: mean = sum / n
            }
        }
        if (masked && masked[c]) s = -9999.0f;
        scores[(size_t)r * C + c] = s;
        if (prob) {
            const float p = iou ? sqrtf(sigmoidf_(s) * iou_s) : sigmoidf_(s);
            prob[(size_t)r * C + c] = p;
            if (p > best || (p == best && c < barg)) { best = p; barg = c; }
        }
    }
    if (!prob || !row_max) return;
    // block arg-max (first index among equals, like torch.max on CPU/CUDA for the documented "first occurrence" case)
    __shared__ float sv[32];
    __shared__ int si[32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, barg, o);
        if (ov > best || (ov == best && oi < barg)) { best = ov; barg = oi; }
    }
    if (lane == 0) { sv[warp] = best; si[warp] = barg; }
    __syncthreads();
    if (warp == 0) {
        const int nw = (blockDim.x + 31) >> 5;
        best = lane < nw ? sv[lane] : -FLT_MAX;
        barg = lane < nw ? si[lane] : 0x7fffffff;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, best, o);
            const int oi = __shfl_xor_sync(0xffffffffu, barg, o);
            if (ov > best || (ov == best && oi < barg)) { best = ov; barg = oi; }
        }
        if (lane == 0) { row_max[r] = best; row_arg[r] = barg; }
    }
}

// ---- in-CTA bitonic sort of (key desc, index asc) pairs held in shared memory; n2 = power of two >= n -------------------
__device__ __forceinline__ bool before(float ka, int ia, float kb, int ib) { return ka > kb || (ka == kb && ia < ib); }

__device__ void bitonic_sort_desc(float* key, int* idx, int n2) {
    for (int k = 2; k <= n2; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < n2; i += blockDim.x) {
                const int l = i ^ j;
                if (l > i) {
                    const bool up = (i & k) == 0;      // ascending position order == "before" order
                    const bool sw = up ? before(key[l], idx[l], key[i], idx[i]) : before(key[i], idx[i], key[l], idx[l]);
                    if (sw) {
                        const float tk = key[i]; key[i] = key[l]; key[l] = tk;
                        const int ti = idx[i]; idx[i] = idx[l]; idx[l] = ti;
                    }
                }
            }
            __syncthreads();
        }
    }
}

// shared memory of batched_nms_kernel for N boxes: sort keys and indices, offset boxes, the N x N pair bit matrix, removed bits
constexpr int nms_smem_bytes(int N) {
    int n2 = 4;
    while (n2 < N) n2 <<= 1;
    const int words = (N + 31) / 32;
    return n2 * 8 + N * 16 + N * words * 4 + words * 4 + 64;
}
constexpr int NMS_SMEM_CAP = 220 * 1024;
constexpr int NMS_MAX = 1216;     // boxes per image (HIPIE: 900): the largest N whose pair matrix fits NMS_SMEM_CAP
static_assert(nms_smem_bytes(NMS_MAX) <= NMS_SMEM_CAP && nms_smem_bytes(NMS_MAX + 1) > NMS_SMEM_CAP, "NMS_MAX is the shared-memory limit");

// boxes (B, N, 4) cxcywh normalised | scores (B, N) | cls (B, N) int32 -> keep (B, N) int32 kept indices in decreasing score
// order (-1 padded), nkeep (B)
__global__ void __launch_bounds__(1024) batched_nms_kernel(const float* __restrict__ boxes, const float* __restrict__ scores,
                                                           const int* __restrict__ cls, int* __restrict__ keep, int* __restrict__ nkeep,
                                                           int N, float thr) {
    extern __shared__ __align__(16) unsigned char nms_smem[];
    const int b = blockIdx.x;
    int n2 = 4;                                   // >= 4 keeps the float4 array behind key/idx 16-byte aligned
    while (n2 < N) n2 <<= 1;
    const int words = (N + 31) >> 5;
    float* key = reinterpret_cast<float*>(nms_smem);             // [n2]
    int* idx = reinterpret_cast<int*>(key + n2);                 // [n2]
    float4* bx = reinterpret_cast<float4*>(idx + n2);            // [N] offset boxes, sorted order
    uint32_t* mask = reinterpret_cast<uint32_t*>(bx + N);        // [N][words]
    uint32_t* removed = mask + (size_t)N * words;                // [words]
    __shared__ float s_max;
    const float* bb = boxes + (size_t)b * N * 4;
    // max coordinate over the xyxy boxes of this image (torchvision: boxes.max())
    float mx = -FLT_MAX;
    for (int i = threadIdx.x; i < N; i += blockDim.x) {
        const float cx = bb[4 * i], cy = bb[4 * i + 1], w = bb[4 * i + 2], h = bb[4 * i + 3];
        mx = fmaxf(mx, fmaxf(fmaxf(cx - 0.5f * w, cy - 0.5f * h), fmaxf(cx + 0.5f * w, cy + 0.5f * h)));
    }
    mx = warp_max(mx);
    __shared__ float wm[32];
    if ((threadIdx.x & 31) == 0) wm[threadIdx.x >> 5] = mx;
    __syncthreads();
    if (threadIdx.x < 32) {
        float v = threadIdx.x < (blockDim.x >> 5) ? wm[threadIdx.x] : -FLT_MAX;
        v = warp_max(v);
        if (threadIdx.x == 0) s_max = v;
    }
    for (int i = threadIdx.x; i < n2; i += blockDim.x) {
        key[i] = i < N ? scores[(size_t)b * N + i] : -FLT_MAX;
        idx[i] = i < N ? i : 0x7fffffff;
    }
    __syncthreads();
    bitonic_sort_desc(key, idx, n2);
    const float off1 = s_max + 1.0f;
    for (int i = threadIdx.x; i < N; i += blockDim.x) {
        const int s = idx[i];
        const float cx = bb[4 * s], cy = bb[4 * s + 1], w = bb[4 * s + 2], h = bb[4 * s + 3];
        // offsets = idxs.to(boxes) * (max_coordinate + 1), rounded before the add as torchvision's tensors are: a contracted
        // cls * off1 + x (one FMA) moves the boxes of class ids in the hundreds by up to 6e-5 at coordinates ~1700
        const float o = __fmul_rn((float)cls[(size_t)b * N + s], off1);
        bx[i] = make_float4((cx - 0.5f * w) + o, (cy - 0.5f * h) + o, (cx + 0.5f * w) + o, (cy + 0.5f * h) + o);
    }
    for (int i = threadIdx.x; i < words; i += blockDim.x) removed[i] = 0;
    __syncthreads();
    // pair matrix: bit j of mask[i][.] = box j (j > i in sorted order) overlaps box i by more than thr
    for (int t = threadIdx.x; t < N * words; t += blockDim.x) {
        const int i = t / words, wj = t - i * words;
        uint32_t m = 0;
        const float4 a = bx[i];
        const float sa = __fmul_rn(a.z - a.x, a.w - a.y);      // areas and intersection rounded as torchvision's (no FMA into the sum)
        const int j0 = wj * 32;
        if (j0 + 31 > i) {
            for (int jj = 0; jj < 32; ++jj) {
                const int j = j0 + jj;
                if (j > i && j < N) {
                    const float4 c = bx[j];
                    const float left = fmaxf(a.x, c.x), right = fminf(a.z, c.z);
                    const float top = fmaxf(a.y, c.y), bottom = fminf(a.w, c.w);
                    const float width = fmaxf(right - left, 0.f), height = fmaxf(bottom - top, 0.f);
                    const float inter = __fmul_rn(width, height);
                    const float sb = __fmul_rn(c.z - c.x, c.w - c.y);
                    if (inter / (sa + sb - inter) > thr) m |= 1u << jj;
                }
            }
        }
        mask[t] = m;
    }
    __syncthreads();
    if (threadIdx.x < 32) {
        int nk = 0;
        for (int i = 0; i < N; ++i) {
            const uint32_t r = removed[i >> 5];         // uniform read
            if (!((r >> (i & 31)) & 1u)) {
                if (threadIdx.x == 0) keep[(size_t)b * N + nk] = idx[i];
                ++nk;
                for (int wj = threadIdx.x; wj < words; wj += 32) removed[wj] |= mask[(size_t)i * words + wj];
            }
            __syncwarp();
        }
        for (int i = nk + threadIdx.x; i < N; i += 32) keep[(size_t)b * N + i] = -1;
        if (threadIdx.x == 0) nkeep[b] = nk;
    }
}

// order-preserving map float -> uint32 (larger float = larger integer); NaNs sort above +inf like torch.topk treats them as largest
__device__ __forceinline__ uint32_t fkey(float v) {
    const uint32_t u = __float_as_uint(v);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

constexpr int TOPK_MAXK = 1024;

// values: row r at values + r * row_stride, n_valid[r] (or n) elements -> out_val (R, k), out_idx (R, k); rows shorter than k are
// padded with (-inf, -1).  Optional gather: `rows` (R,) int32 list of source rows is not needed -- callers pass compacted input.
__global__ void __launch_bounds__(1024) topk_kernel(const float* __restrict__ values, int64_t row_stride, const int* __restrict__ n_rows,
                                                    int n_cols_per_row, int n, int k, float* __restrict__ out_val,
                                                    int* __restrict__ out_idx) {
    __shared__ uint32_t hist[256];
    __shared__ uint32_t s_prefix, s_remaining, s_count;
    __shared__ float ckey[2 * TOPK_MAXK];
    __shared__ int cidx[2 * TOPK_MAXK];
    const int r = blockIdx.x;
    const float* v = values + (size_t)r * row_stride;
    const int len = n_rows ? min(n, n_rows[r] * n_cols_per_row) : n;
    const int kk = min(k, len);
    float* ov = out_val + (size_t)r * k;
    int* oi = out_idx + (size_t)r * k;
    if (kk <= 0) {
        for (int i = threadIdx.x; i < k; i += blockDim.x) { ov[i] = -INFINITY; oi[i] = -1; }
        return;
    }
    // ---- radix select of the kk-th largest key, most significant byte first
    if (threadIdx.x == 0) { s_prefix = 0; s_remaining = (uint32_t)kk; }
    __syncthreads();
    for (int pass = 0; pass < 4; ++pass) {
        const int shift = 24 - 8 * pass;
        for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0;
        __syncthreads();
        const uint32_t prefix = s_prefix;
        const uint32_t pmask = pass == 0 ? 0u : (0xffffffffu << (shift + 8));
        for (int i = threadIdx.x; i < len; i += blockDim.x) {
            const uint32_t key = fkey(v[i]);
            if ((key & pmask) == prefix) atomicAdd(&hist[(key >> shift) & 255u], 1u);
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            uint32_t rem = s_remaining;
            int d = 255;
            for (; d > 0; --d) {
                if (hist[d] >= rem) break;
                rem -= hist[d];
            }
            s_prefix = prefix | ((uint32_t)d << shift);
            s_remaining = rem;                       // how many of the elements equal to the threshold digit path are still needed
        }
        __syncthreads();
    }
    const uint32_t tkey = s_prefix;                  // key of the kk-th largest element
    // ---- collect: everything strictly above the threshold, plus threshold-equal elements in index order until kk is reached.
    //      Strictly-above count is kk - s_remaining; equal elements fill the rest (lowest index first: deterministic).
    if (threadIdx.x == 0) s_count = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < len; i += blockDim.x) {
        const float x = v[i];
        if (fkey(x) > tkey) {
            const uint32_t p = atomicAdd(&s_count, 1u);
            if (p < 2 * TOPK_MAXK) { ckey[p] = x; cidx[p] = i; }
        }
    }
    __syncthreads();
    const uint32_t above = s_count;
    // equal-to-threshold elements: ordered by index.  One warp walks the row in index order with a ballot prefix.
    if (threadIdx.x < 32) {
        uint32_t need = (uint32_t)kk - above, got = 0;
        for (int base = 0; base < len && got < need; base += 32) {
            const int i = base + threadIdx.x;
            const bool eq = i < len && fkey(v[i]) == tkey;
            const uint32_t bal = __ballot_sync(0xffffffffu, eq);
            const uint32_t rank = got + __popc(bal & ((1u << threadIdx.x) - 1u));
            if (eq && rank < need) { ckey[above + rank] = v[i]; cidx[above + rank] = i; }
            got += __popc(bal);
        }
    }
    __syncthreads();
    int n2 = 1;
    while (n2 < kk) n2 <<= 1;
    for (int i = kk + threadIdx.x; i < n2; i += blockDim.x) { ckey[i] = -INFINITY; cidx[i] = 0x7fffffff; }
    __syncthreads();
    bitonic_sort_desc(ckey, cidx, n2);
    for (int i = threadIdx.x; i < k; i += blockDim.x) {
        ov[i] = i < kk ? ckey[i] : -INFINITY;
        oi[i] = i < kk ? cidx[i] : -1;
    }
}

}  // namespace

// Greedy NMS over many boxes (the automatic mask generator: 3072 candidates per crop of a 32 x 32 point grid, and all crops together),
// too many for batched_nms_kernel's shared-memory pair matrix.  The boxes come sorted by decreasing score.
//   nms_tile_kernel   grid (tiles, tiles), 64 threads: bit j of mask[i][c] = IoU(box i, box 64 c + j) > thr for 64 c + j > i, as
//                     torchvision's nms (IoU = inter / (area_i + area_j - inter), area = (x2 - x1) * (y2 - y1)); tiles left of the
//                     diagonal are never read and not written
//   nms_sweep_kernel  one CTA: per tile of 64 boxes one thread resolves the tile's own bits in order, then the CTA ORs the rows of the
//                     boxes it kept into the removed bits of the later tiles
constexpr int NMS_TILE = 64, NMS_SORTED_MAX = 32768, NMS_SWEEP_THREADS = 256;

__global__ void __launch_bounds__(NMS_TILE)
nms_tile_kernel(const float* __restrict__ boxes, int N, float thr, int tiles, unsigned long long* __restrict__ mask) {
    const int rt = blockIdx.y, ct = blockIdx.x;
    if (ct < rt) return;
    __shared__ float4 cb[NMS_TILE];
    const int nc = min(NMS_TILE, N - ct * NMS_TILE), j0 = ct * NMS_TILE;
    if ((int)threadIdx.x < nc) cb[threadIdx.x] = reinterpret_cast<const float4*>(boxes)[j0 + threadIdx.x];
    __syncthreads();
    const int i = rt * NMS_TILE + threadIdx.x;
    if (i >= N) return;
    const float4 a = reinterpret_cast<const float4*>(boxes)[i];
    const float sa = (a.z - a.x) * (a.w - a.y);
    unsigned long long bits = 0;
    for (int j = rt == ct ? (int)threadIdx.x + 1 : 0; j < nc; ++j) {
        const float4 c = cb[j];
        const float width = fmaxf(fminf(a.z, c.z) - fmaxf(a.x, c.x), 0.f), height = fmaxf(fminf(a.w, c.w) - fmaxf(a.y, c.y), 0.f);
        const float inter = width * height;
        const float sb = (c.z - c.x) * (c.w - c.y);
        if (inter / (sa + sb - inter) > thr) bits |= 1ull << j;
    }
    mask[(int64_t)i * tiles + ct] = bits;
}

__global__ void __launch_bounds__(NMS_SWEEP_THREADS)
nms_sweep_kernel(const unsigned long long* __restrict__ mask, int N, int tiles, int* __restrict__ keep, int* __restrict__ nkeep) {
    extern __shared__ unsigned long long removed[];              // [tiles]
    __shared__ unsigned long long diag[NMS_TILE];
    __shared__ int kept[NMS_TILE];
    __shared__ int s_nb;
    for (int t = threadIdx.x; t < tiles; t += NMS_SWEEP_THREADS) removed[t] = 0;
    int nk = 0;                                                  // thread 0's count of kept boxes
    for (int t = 0; t < tiles; ++t) {
        const int rows = min(NMS_TILE, N - t * NMS_TILE);
        __syncthreads();
        if ((int)threadIdx.x < rows) diag[threadIdx.x] = mask[(int64_t)(t * NMS_TILE + threadIdx.x) * tiles + t];
        __syncthreads();
        if (threadIdx.x == 0) {
            unsigned long long cur = removed[t];
            int nb = 0;
            for (int r = 0; r < rows; ++r) {
                if (!((cur >> r) & 1ull)) {
                    kept[nb++] = t * NMS_TILE + r;
                    keep[nk++] = t * NMS_TILE + r;
                    cur |= diag[r];
                }
            }
            s_nb = nb;
        }
        __syncthreads();
        const int nb = s_nb;
        for (int c = t + 1 + threadIdx.x; c < tiles; c += NMS_SWEEP_THREADS) {
            unsigned long long acc = removed[c];
            for (int r = 0; r < nb; ++r) acc |= mask[(int64_t)kept[r] * tiles + c];
            removed[c] = acc;
        }
    }
    if (threadIdx.x == 0) *nkeep = nk;
}

}  // namespace hipie

using namespace hipie;

extern "C" int hipie_class_scores(const float* logits, const int* tok, const int* cnt, const int8_t* masked, const float* iou,
                                  float* scores, float* prob, float* row_max, int* row_arg, int R, int Lt, int C, int maxlen,
                                  int max_pool, void* stream) {
    HIPIE_CHECK_ARG(logits && tok && cnt && scores, "hipie_class_scores: null pointer argument");
    HIPIE_CHECK_ARG(R >= 0 && Lt > 0 && C > 0 && maxlen > 0, "hipie_class_scores: bad sizes R=%d Lt=%d C=%d maxlen=%d", R, Lt, C, maxlen);
    HIPIE_CHECK_ARG(!row_max || (prob && row_arg), "hipie_class_scores: row_max needs prob and row_arg");
    if (R == 0) return HIPIE_OK;
    const int threads = C >= 256 ? 256 : (C >= 128 ? 128 : 64);
    class_scores_kernel<<<R, threads, 0, (cudaStream_t)stream>>>(logits, tok, cnt, masked, iou, scores, prob, row_max, row_arg, R, Lt, C,
                                                                 maxlen, max_pool);
    HIPIE_CHECK_LAUNCH();
    return HIPIE_OK;
}

extern "C" int hipie_batched_nms(const float* boxes_cxcywh, const float* scores, const int* cls, int* keep, int* nkeep, int B, int N,
                                 float iou_threshold, void* stream) {
    HIPIE_CHECK_ARG(boxes_cxcywh && scores && cls && keep && nkeep, "hipie_batched_nms: null pointer argument");
    HIPIE_CHECK_ARG(B >= 0 && N > 0 && N <= NMS_MAX, "hipie_batched_nms: N=%d outside (0, %d]", N, NMS_MAX);
    if (B == 0) return HIPIE_OK;
    const int smem = nms_smem_bytes(N);
    HIPIE_ENSURE_SMEM(batched_nms_kernel, smem);
    batched_nms_kernel<<<B, 1024, smem, (cudaStream_t)stream>>>(boxes_cxcywh, scores, cls, keep, nkeep, N, iou_threshold);
    HIPIE_CHECK_LAUNCH();
    return HIPIE_OK;
}

extern "C" int hipie_topk(const float* values, int64_t row_stride, const int* n_rows, int n_cols_per_row, int R, int n, int k,
                          float* out_val, int* out_idx, void* stream) {
    HIPIE_CHECK_ARG(values && out_val && out_idx, "hipie_topk: null pointer argument");
    HIPIE_CHECK_ARG(R >= 0 && n > 0 && k > 0 && k <= TOPK_MAXK, "hipie_topk: bad sizes R=%d n=%d k=%d (k <= %d)", R, n, k, TOPK_MAXK);
    if (R == 0) return HIPIE_OK;
    topk_kernel<<<R, 1024, 0, (cudaStream_t)stream>>>(values, row_stride, n_rows, n_cols_per_row, n, k, out_val, out_idx);
    HIPIE_CHECK_LAUNCH();
    return HIPIE_OK;
}

extern "C" int hipie_nms_sorted(const float* boxes_xyxy, int N, float iou_threshold, unsigned long long* mask_ws, int64_t ws_words,
                                int* keep, int* nkeep, void* stream) {
    HIPIE_CHECK_ARG(nkeep && (N == 0 || (boxes_xyxy && mask_ws && keep)), "hipie_nms_sorted: null pointer argument");
    HIPIE_CHECK_ARG(N >= 0 && N <= NMS_SORTED_MAX, "hipie_nms_sorted: N=%d outside [0, %d]", N, NMS_SORTED_MAX);
    HIPIE_CHECK_ARG((reinterpret_cast<uintptr_t>(boxes_xyxy) & 15) == 0, "hipie_nms_sorted: boxes must be 16-byte aligned");
    const int tiles = (N + NMS_TILE - 1) / NMS_TILE;
    HIPIE_CHECK_ARG(ws_words >= (int64_t)N * tiles, "hipie_nms_sorted: workspace of %lld words < N * ceil(N / 64) = %lld",
                    (long long)ws_words, (long long)N * tiles);
    cudaStream_t st = (cudaStream_t)stream;
    if (N == 0) {
        HIPIE_CHECK_CUDA(cudaMemsetAsync(nkeep, 0, sizeof(int), st));
        return HIPIE_OK;
    }
    nms_tile_kernel<<<dim3(tiles, tiles), NMS_TILE, 0, st>>>(boxes_xyxy, N, iou_threshold, tiles, mask_ws);
    HIPIE_CHECK_LAUNCH();
    nms_sweep_kernel<<<1, NMS_SWEEP_THREADS, tiles * sizeof(unsigned long long), st>>>(mask_ws, N, tiles, keep, nkeep);
    HIPIE_CHECK_LAUNCH();
    return HIPIE_OK;
}
