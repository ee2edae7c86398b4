// Fused semantic + panoptic post-processing (SURVEY.md §8 rows a22/a23; reference H/models/hipie_img.py:880-1023).
//
// The reference upsamples every query's 1/4-resolution mask logit to full resolution (bilinear, align_corners=False),
// takes the sigmoid, and then (a) contracts it with the per-query class probabilities into a (C, H, W) semantic map
// (einsum "qc,qhw->chw") and (b) takes an argmax over score*sigmoid for the kept queries plus three per-query pixel
// counts for the panoptic merge.  As separate ops that is Q*H*W fp32 written and re-read four times (~5 GB per image at
// Q=1200, 1024^2).  Here one kernel does it all from the low-resolution logits: each CTA owns a 32x8 pixel tile, stages
// the 9x3 low-resolution taps of 64 queries at a time in shared memory, evaluates sigmoid(bilinear()) straight into
// mma.sync A fragments (bf16 hi/lo split), and accumulates the (pixels x classes) tile on the tensor cores in bf16x3
// against the class-probability chunk; the argmax / area counters ride along on the same sigmoid values.
// HBM traffic drops to the low-resolution logits (+halo) and the outputs.
#include "common.cuh"
#include <algorithm>
#include <stdlib.h>

namespace hipie {

namespace {

constexpr int PP_BX = 8, PP_BY = 2;           // 4x4-pixel blocks per CTA (x, y): a 32x8 pixel tile, shifted by (-2,-2)
constexpr int PP_QC = 64;                     // queries per staged chunk
constexpr int PP_TR = PP_BY + 1, PP_TC = PP_BX + 1;   // low-resolution rows / cols a tile touches
constexpr int PP_TQ = PP_TR * PP_TC;          // floats per query in the tap tile (27: odd stride, conflict-free across t)
constexpr int PP_PQ = PP_QC + 8;              // padded bf16 per class row of the staged P^T chunk
constexpr int PP_THREADS = 256;
constexpr int PP_NLD = (PP_QC * PP_TQ + PP_THREADS - 1) / PP_THREADS;   // tap loads per thread per chunk

__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ float rcp_approx(float x) {
    float y;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(smem)), "l"(gmem));
}

// With stride 4 and align_corners=False every aligned 4x4 pixel block [4k-2, 4k+2) shares its four low-resolution taps
// (columns k-1,k; clamping the tap index reproduces the border rule) and the weights are the constants 1/8,3/8,5/8,7/8.
// One m16 MMA tile is one such block, so a thread reads 4 taps per (block, query) for its two pixels.
//
// masks (Q,h,w) f32 | pt_hi/pt_lo (NT*8, Qpad) bf16 = class probabilities transposed, split | scores (Qpad) f32, 0 = not kept
// sem (C,Hc,Wc) f32 | ids (Hc,Wc) i32 = -1 or 2*q + (sigmoid_q >= .5) | areas (3,Q) i32 = mask / original / intersection
template <int NT>
__global__ void __launch_bounds__(PP_THREADS, NT <= 10 ? 2 : 1)
seg_post_kernel(const float* __restrict__ masks, const __nv_bfloat16* __restrict__ pt_hi,
                const __nv_bfloat16* __restrict__ pt_lo, const float* __restrict__ scores, float* __restrict__ sem,
                int* __restrict__ ids, int* __restrict__ areas, int Q, int Qpad, int C, int h, int w, int Hc, int Wc) {
    extern __shared__ __align__(16) unsigned char pp_smem[];
    constexpr int P_ELEMS = NT * 8 * PP_PQ;
    static_assert((PP_QC * PP_TQ * 4 * 2) % 16 == 0, "P^T chunk must stay 16-byte aligned");
    float* taps = reinterpret_cast<float*>(pp_smem);                                   // [2][PP_QC][PP_TQ]
    __nv_bfloat16* pbuf = reinterpret_cast<__nv_bfloat16*>(taps + 2 * PP_QC * PP_TQ); // [2][hi,lo][NT*8][PP_PQ]
    float* sc = reinterpret_cast<float*>(pbuf + 4 * P_ELEMS);                          // [2][PP_QC]
    int* cnt = reinterpret_cast<int*>(sc + 2 * PP_QC);                                 // [3][Qpad]

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
    const int kx0 = blockIdx.x * PP_BX, ky0 = blockIdx.y * PP_BY;       // first 4x4 block of this CTA
    const int x_lo = kx0 - 1, y_lo = ky0 - 1;                           // first low-resolution column / row staged

    __shared__ int s_first;              // first kept query (argmax fallback), INT_MAX if none
    if (tid == 0) s_first = 0x7fffffff;
    for (int i = tid; i < 3 * Qpad; i += PP_THREADS) cnt[i] = 0;
    __syncthreads();
    for (int i = tid; i < Q; i += PP_THREADS)
        if (scores[i] > 0.f) atomicMin(&s_first, i);

    // ---- chunk-invariant staging offsets -----------------------------------------------------------------------
    int goff[PP_NLD];
#pragma unroll
    for (int k = 0; k < PP_NLD; ++k) {
        const int idx = tid + k * PP_THREADS;
        const int ql = idx / PP_TQ, rc = idx - ql * PP_TQ;
        const int r = rc / PP_TC, c = rc - r * PP_TC;
        const int yy = min(max(y_lo + r, 0), h - 1), xx = min(max(x_lo + c, 0), w - 1);
        goff[k] = idx < PP_QC * PP_TQ ? (ql * h + yy) * w + xx : -1;
    }
    const size_t hw = (size_t)h * w;
    float tv[PP_NLD];
    auto load_taps = [&](int q0) {
#pragma unroll
        for (int k = 0; k < PP_NLD; ++k) {
            const int ql = (tid + k * PP_THREADS) / PP_TQ;
            // staged as -log2(e) * logit, so sigmoid = 1 / (1 + 2^tap); padding -> +big -> sigmoid 0
            tv[k] = (goff[k] >= 0 && q0 + ql < Q) ? -1.4426950408889634f * __ldg(masks + (size_t)q0 * hw + goff[k]) : 1e30f;
        }
    };
    auto store_taps = [&](int buf) {
#pragma unroll
        for (int k = 0; k < PP_NLD; ++k) {
            const int idx = tid + k * PP_THREADS;
            if (idx < PP_QC * PP_TQ) taps[buf * PP_QC * PP_TQ + idx] = tv[k];
        }
    };
    auto load_p = [&](int q0, int buf) {
        __nv_bfloat16* ph = pbuf + buf * 2 * P_ELEMS;
        for (int i = tid; i < NT * 8 * (PP_QC / 8); i += PP_THREADS) {
            const int row = i / (PP_QC / 8), seg = i - row * (PP_QC / 8);
            cp_async16(ph + row * PP_PQ + seg * 8, pt_hi + (size_t)row * Qpad + q0 + seg * 8);
            cp_async16(ph + P_ELEMS + row * PP_PQ + seg * 8, pt_lo + (size_t)row * Qpad + q0 + seg * 8);
        }
        if (tid < PP_QC / 4) cp_async16(sc + buf * PP_QC + tid * 4, scores + q0 + tid * 4);
        asm volatile("cp.async.commit_group;" ::: "memory");
    };

    // ---- this thread's pixels: blocks (2*(warp&3)+mt, warp>>2), rows dy and dy+2 of the block, column dx --------
    const int dy = g >> 2, dx = g & 3;
    const int kyl = warp >> 2;
    const int y_a = 4 * (ky0 + kyl) - 2 + dy, y_b = y_a + 2;
    const float lx1 = 0.125f + 0.25f * dx, lx0 = 1.f - lx1;
    const float lya1 = 0.125f + 0.25f * dy, lya0 = 1.f - lya1;           // row dy
    const float lyb1 = lya1 + 0.5f, lyb0 = 1.f - lyb1;                   // row dy + 2
    int tb[2], px[2];
    bool pv[4];                                                          // [2*mt + half]
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
        const int kxl = 2 * (warp & 3) + mt;
        tb[mt] = kyl * PP_TC + kxl;
        px[mt] = 4 * (kx0 + kxl) - 2 + dx;
        const bool xv = px[mt] >= 0 && px[mt] < Wc;
        pv[2 * mt] = xv && y_a >= 0 && y_a < Hc;
        pv[2 * mt + 1] = xv && y_b >= 0 && y_b < Hc;
    }

    float acc[2][NT][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < NT; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[mt][nt][e] = 0.f;
    float best[4];                       // running max of score * sigmoid over the kept queries (strictly positive wins)
    int bidx[4];
#pragma unroll
    for (int ps = 0; ps < 4; ++ps) {
        best[ps] = 0.f;
        bidx[ps] = -1;
    }
    // ldmatrix lane address inside a P^T chunk: matrices {hi k0-7, hi k8-15, lo k0-7, lo k8-15} of one 8-class tile
    const int lm_off = ((lane >> 4) ? P_ELEMS : 0) + (lane & 7) * PP_PQ + ((lane >> 3) & 1) * 8;

    load_taps(0);
    load_p(0, 0);
    const int nchunk = Qpad / PP_QC;
    for (int ch = 0; ch < nchunk; ++ch) {
        const int buf = ch & 1, q0 = ch * PP_QC;
        store_taps(buf);
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        __syncthreads();                     // chunk ch staged; everyone is done reading buffers buf^1 (chunk ch-1)
        if (ch + 1 < nchunk) {
            load_taps(q0 + PP_QC);           // in flight during the compute below
            load_p(q0 + PP_QC, buf ^ 1);
        }
        const float* tp = taps + buf * PP_QC * PP_TQ;
        const uint32_t p_addr = (uint32_t)__cvta_generic_to_shared(pbuf + buf * 2 * P_ELEMS + lm_off);
        const float* scb = sc + buf * PP_QC;

#pragma unroll 1
        for (int ks = 0; ks < PP_QC / 16; ++ks) {
            uint32_t ah[2][4], al[2][4];
            uint32_t npack = 0;                       // per-query counts of sigmoid >= .5 over this thread's pixels (8 bits each)
#pragma unroll
            for (int jp = 0; jp < 2; ++jp) {
                float sg[4][2];                       // [ps][j&1]  sigmoid(upsampled logit)
#pragma unroll
                for (int jj = 0; jj < 2; ++jj) {
                    const int j = 2 * jp + jj;
                    const int ql = ks * 16 + 2 * t + jj + jp * 8;
                    const float s_q = scb[ql];        // 0 for queries that are not kept
                    uint32_t n = 0;
#pragma unroll
                    for (int mt = 0; mt < 2; ++mt) {
                        const float* T = tp + ql * PP_TQ + tb[mt];
                        const float t00 = T[0], t10 = T[PP_TC];
                        const float top = fmaf(lx1, T[1] - t00, t00);
                        const float bot = fmaf(lx1, T[PP_TC + 1] - t10, t10);
                        const float d = bot - top;
#pragma unroll
                        for (int half = 0; half < 2; ++half) {
                            const int ps = 2 * mt + half;
                            const float v = fmaf(half ? lyb1 : lya1, d, top);       // -log2(e) * upsampled logit
                            const float s = rcp_approx(1.f + ex2_approx(v));
                            sg[ps][jj] = s;
                            const float pr = s * s_q;
                            const bool up = pr > best[ps];
                            best[ps] = up ? pr : best[ps];
                            bidx[ps] = up ? q0 + ql : bidx[ps];
                            n += (pv[ps] && v <= 0.f) ? 1u : 0u;                    // sigmoid >= .5  <=>  logit >= 0
                        }
                    }
                    npack |= n << (8 * j);
                }
#pragma unroll
                for (int mt = 0; mt < 2; ++mt) {
                    split2(sg[2 * mt][0], sg[2 * mt][1], ah[mt][2 * jp], al[mt][2 * jp]);
                    split2(sg[2 * mt + 1][0], sg[2 * mt + 1][1], ah[mt][2 * jp + 1], al[mt][2 * jp + 1]);
                }
            }
            // counts: sum over the 8 pixel lanes that share t, then lane g = j adds the byte of query slot j
            npack += __shfl_xor_sync(0xffffffffu, npack, 4);
            npack += __shfl_xor_sync(0xffffffffu, npack, 8);
            npack += __shfl_xor_sync(0xffffffffu, npack, 16);
            if (g < 4) {
                const uint32_t n = (npack >> (8 * g)) & 0xffu;
                if (n) atomicAdd(&cnt[Qpad + q0 + ks * 16 + 2 * t + (g & 1) + (g >> 1) * 8], (int)n);
            }
#pragma unroll
            for (int nt = 0; nt < NT; ++nt) {
                uint32_t bh0, bh1, bl0, bl1;
                asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                             : "=r"(bh0), "=r"(bh1), "=r"(bl0), "=r"(bl1)
                             : "r"(p_addr + (uint32_t)((nt * 8 * PP_PQ + ks * 16) * 2)));
                mma16816(acc[0][nt], ah[0], bh0, bh1);
                mma16816(acc[1][nt], ah[1], bh0, bh1);
                mma16816(acc[0][nt], ah[0], bl0, bl1);
                mma16816(acc[1][nt], ah[1], bl0, bl1);
                mma16816(acc[0][nt], al[0], bh0, bh1);
                mma16816(acc[1][nt], al[1], bh0, bh1);
            }
        }
    }

    // ---- argmax across the quad (ties -> lowest query index, like torch.argmax over the kept list) -------------
    // A pixel where every kept query has score*sigmoid == 0 (sigmoid underflow) goes to the first kept query, as argmax would.
#pragma unroll
    for (int ps = 0; ps < 4; ++ps) {
#pragma unroll
        for (int o = 1; o <= 2; o <<= 1) {
            const float ob = __shfl_xor_sync(0xffffffffu, best[ps], o);
            const int oi = __shfl_xor_sync(0xffffffffu, bidx[ps], o);
            const bool take = (oi >= 0) && (bidx[ps] < 0 || ob > best[ps] || (ob == best[ps] && oi < bidx[ps]));
            if (take) {
                best[ps] = ob;
                bidx[ps] = oi;
            }
        }
        if (t == 0 && pv[ps]) {
            const int y = (ps & 1) ? y_b : y_a;
            int bi = bidx[ps], in = 0;
            if (bi >= 0) in = best[ps] >= 0.5f * scores[bi];      // sigmoid >= .5 for the winner
            else bi = s_first == 0x7fffffff ? -1 : s_first;
            ids[(size_t)y * Wc + px[ps >> 1]] = bi < 0 ? -1 : 2 * bi + in;
            if (bi >= 0) {
                atomicAdd(&cnt[bi], 1);
                if (in) atomicAdd(&cnt[2 * Qpad + bi], 1);
            }
        }
    }
    // ---- semantic tile ------------------------------------------------------------------------------------------
    const size_t plane = (size_t)Hc * Wc;
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < NT; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int ps = 2 * mt + (e >> 1);
                const int c = nt * 8 + 2 * t + (e & 1);
                const int y = (e >> 1) ? y_b : y_a;
                if (pv[ps] && c < C) sem[c * plane + (size_t)y * Wc + px[mt]] = acc[mt][nt][e];
            }
    __syncthreads();
    for (int i = tid; i < 3 * Qpad; i += PP_THREADS) {
        const int v = cnt[i];
        const int a = i / Qpad, q = i - a * Qpad;
        if (v && q < Q) atomicAdd(&areas[a * Q + q], v);
    }
}

}  // namespace
}  // namespace hipie
namespace hipie {
namespace {

// Instance masks (hipie_img.py:1003-1007): bilinear x4 (align_corners=False) of the 1/4-resolution logits, sigmoid, > threshold,
// crop -- one pass, one byte per pixel out.  Thread = 4 consecutive pixels of one 4x4 block row (they share the 4 taps).
__global__ void __launch_bounds__(256)
upsample_threshold_kernel(const float* __restrict__ masks, uint8_t* __restrict__ out, int N, int h, int w, int Hc, int Wc,
                          float thr) {
    const int kxn = (Wc + 2 + 3) / 4;                       // 4-pixel groups [4k-2, 4k+2) per row
    const int64_t total = (int64_t)N * Hc * kxn;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int kx = (int)(i % kxn);
        const int y = (int)((i / kxn) % Hc);
        const int n = (int)(i / ((int64_t)kxn * Hc));
        const float sy = fmaxf(0.25f * (y + 0.5f) - 0.5f, 0.f);
        const int y0 = min((int)sy, h - 1), y1 = y0 + (y0 < h - 1);
        const float ly = sy - y0;
        const int x0 = max(kx - 1, 0), x1 = min(kx, w - 1);
        const float* m0 = masks + ((int64_t)n * h + y0) * w;
        const float* m1 = masks + ((int64_t)n * h + y1) * w;
        const float t00 = __ldg(m0 + x0), t01 = __ldg(m0 + x1), t10 = __ldg(m1 + x0), t11 = __ldg(m1 + x1);
#pragma unroll
        for (int dx = 0; dx < 4; ++dx) {
            const int x = 4 * kx - 2 + dx;
            if (x < 0 || x >= Wc) continue;
            // same expression order as upsample_bilinear2d: h0*(w0*a + w1*b) + h1*(w0*c + w1*d)
            float lx = 0.125f + 0.25f * dx;
            if (kx == 0) lx = 0.f;                          // clamped source index at the left border
            const float v = (1.f - ly) * ((1.f - lx) * t00 + lx * t01) + ly * ((1.f - lx) * t10 + lx * t11);
            const float sg = 1.f / (1.f + expf(-v));
            out[((int64_t)n * Hc + y) * Wc + x] = sg > thr ? 1 : 0;
        }
    }
}

template <int NT>
int launch_seg_post(const float* masks, const void* pt_hi, const void* pt_lo, const float* scores, float* sem, int* ids,
                    int* areas, int Q, int Qpad, int C, int h, int w, int Hc, int Wc, cudaStream_t st) {
    const int smem = 2 * PP_QC * PP_TQ * 4 + 4 * NT * 8 * PP_PQ * 2 + 2 * PP_QC * 4 + 3 * Qpad * 4;
    HIPIE_CHECK_ARG(smem <= 220 * 1024, "hipie_seg_postprocess: Q=%d needs %d B of shared memory", Q, smem);
    HIPIE_ENSURE_SMEM(seg_post_kernel<NT>, smem);
    dim3 grid(((Wc + 2 + 3) / 4 + PP_BX - 1) / PP_BX, ((Hc + 2 + 3) / 4 + PP_BY - 1) / PP_BY);
    seg_post_kernel<NT><<<grid, PP_THREADS, smem, st>>>(masks, (const __nv_bfloat16*)pt_hi, (const __nv_bfloat16*)pt_lo, scores,
                                                       sem, ids, areas, Q, Qpad, C, h, w, Hc, Wc);
    HIPIE_CHECK_LAUNCH();
    return HIPIE_OK;
}

}  // namespace
}  // namespace hipie

using namespace hipie;

extern "C" int hipie_seg_postprocess(const float* masks, const void* pt_hi, const void* pt_lo, const float* scores,
                                     float* sem, int* ids, int* areas, int Q, int Qpad, int C, int h, int w, int stride,
                                     int Hc, int Wc, void* stream) {
    HIPIE_CHECK_ARG(masks && pt_hi && pt_lo && scores && sem && ids && areas, "hipie_seg_postprocess: null pointer");
    HIPIE_CHECK_ARG(stride == 4, "hipie_seg_postprocess: only mask stride 4 is implemented (got %d)", stride);
    HIPIE_CHECK_ARG(Q > 0 && Qpad >= Q && Qpad % PP_QC == 0 && C > 0 && C <= 136 && h > 1 && w > 1 && Hc > 0 && Wc > 0 &&
                        Hc <= 4 * h && Wc <= 4 * w,
                    "hipie_seg_postprocess: bad sizes Q=%d Qpad=%d C=%d h=%d w=%d Hc=%d Wc=%d", Q, Qpad, C, h, w, Hc, Wc);
    HIPIE_CHECK_CUDA(cudaMemsetAsync(areas, 0, sizeof(int) * 3 * Q, (cudaStream_t)stream));
    if (C <= 80)
        return launch_seg_post<10>(masks, pt_hi, pt_lo, scores, sem, ids, areas, Q, Qpad, C, h, w, Hc, Wc, (cudaStream_t)stream);
    return launch_seg_post<17>(masks, pt_hi, pt_lo, scores, sem, ids, areas, Q, Qpad, C, h, w, Hc, Wc, (cudaStream_t)stream);
}

extern "C" int hipie_upsample_threshold(const float* masks, void* out_u8, int N, int h, int w, int stride, int Hc, int Wc,
                                        float threshold, void* stream) {
    if (N == 0) return HIPIE_OK;     // empty detections: nothing to write (pointers of empty tensors may be null)
    HIPIE_CHECK_ARG(masks && out_u8, "hipie_upsample_threshold: null pointer");
    HIPIE_CHECK_ARG(stride == 4, "hipie_upsample_threshold: only mask stride 4 is implemented (got %d)", stride);
    HIPIE_CHECK_ARG(N >= 0 && h > 1 && w > 1 && Hc > 0 && Wc > 0 && Hc <= 4 * h && Wc <= 4 * w,
                    "hipie_upsample_threshold: bad sizes N=%d h=%d w=%d Hc=%d Wc=%d", N, h, w, Hc, Wc);
    const int64_t total = (int64_t)N * Hc * ((Wc + 5) / 4);
    const int blocks = (int)std::min<int64_t>((total + 255) / 256, (int64_t)num_sms() * 32);
    upsample_threshold_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(masks, (uint8_t*)out_u8, N, h, w, Hc, Wc, threshold);
    HIPIE_CHECK_LAUNCH();
    return HIPIE_OK;
}
