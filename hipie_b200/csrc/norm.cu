// LayerNorm / GroupNorm for the hot path (fp32 statistics, fp32 and/or bf16-split outputs so the
// normalised activations feed the wgmma GEMM without a separate conversion pass).
// Reference call sites: ViT pre-LN eps 1e-6 (/root/reference/projects/HIPIE/hipie/backbone/vit.py:212-230),
// DETR / MaskDINO post-LN eps 1e-5 (deformable_transformer_dino.py:385-450), GroupNorm(32) of the
// input projections (deformable_detr.py:221-236, maskdino_encoder.py:253-306).
#include "common.cuh"
#include "ptx.cuh"

namespace hipie {

// one warp per row, C % 128 == 0, C <= 128*MAXV
template <int MAXV>
__global__ void __launch_bounds__(256)
layernorm_kernel(const float* __restrict__ x, const float* __restrict__ add, const float* __restrict__ gamma,
                 const float* __restrict__ beta, float eps, float* __restrict__ sum_out,
                 float* __restrict__ y_f32, __nv_bfloat16* __restrict__ y_hi, __nv_bfloat16* __restrict__ y_lo,
                 int64_t rows, int C, const int* __restrict__ omap, int y_fp16, uint8_t* __restrict__ y8) {
    const int lane = threadIdx.x & 31;
    const int nv = C >> 7;
    // grid-stride over rows: the launcher caps the grid at the number of resident CTAs, so a 32768-row call is one full wave of
    // long-lived CTAs instead of 3.5 waves of 8-row CTAs with a 46 % tail
    const int64_t wstride = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < rows; row += wstride) {
    const int64_t orow = omap ? omap[row] : row;
    const float* xr = x + row * C;
    float4 v[MAXV];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
        if (i < nv) {
            v[i] = *reinterpret_cast<const float4*>(xr + (i * 32 + lane) * 4);
            if (add) {
                const float4 a = *reinterpret_cast<const float4*>(add + row * C + (i * 32 + lane) * 4);
                v[i].x += a.x; v[i].y += a.y; v[i].z += a.z; v[i].w += a.w;
                if (sum_out) *reinterpret_cast<float4*>(sum_out + row * C + (i * 32 + lane) * 4) = v[i];
            }
            s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
        }
    }
    const float mean = warp_sum(s) / (float)C;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
        if (i < nv) {
            const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
            q += (a * a + b * b) + (c * c + d * d);
        }
    }
    const float rstd = rsqrtf(warp_sum(q) / (float)C + eps);
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
        if (i < nv) {
            const int c0 = (i * 32 + lane) * 4;
            const float4 g = *reinterpret_cast<const float4*>(gamma + c0);
            const float4 b = *reinterpret_cast<const float4*>(beta + c0);
            float4 o;
            o.x = (v[i].x - mean) * rstd * g.x + b.x;
            o.y = (v[i].y - mean) * rstd * g.y + b.y;
            o.z = (v[i].z - mean) * rstd * g.z + b.z;
            o.w = (v[i].w - mean) * rstd * g.w + b.w;
            if (y_f32) *reinterpret_cast<float4*>(y_f32 + orow * C + c0) = o;
            if (y_hi && y8) {                                // fp16 plane + e4m3 planes [e4m3(h) | e4m3(2^10 (o - h))] (prec-6 GEMM operand)
                uint2 h16;
                uint32_t a8, b8;
                split4_f16_e4m3(o, h16, a8, b8);
                *reinterpret_cast<uint2*>(y_hi + orow * C + c0) = h16;
                uint8_t* o8 = y8 + orow * 2 * C + e4m3_slot0(c0);
                *reinterpret_cast<uint32_t*>(o8) = a8;
                *reinterpret_cast<uint32_t*>(o8 + 32) = b8;
            } else if (y_hi) {
                uint2 hi, lo;
                split2m(o.x, o.y, hi.x, lo.x, y_fp16);       // y_fp16: y_hi is ONE IEEE fp16 plane (y_lo NULL)
                split2m(o.z, o.w, hi.y, lo.y, y_fp16);
                *reinterpret_cast<uint2*>(y_hi + orow * C + c0) = hi;
                if (y_lo) *reinterpret_cast<uint2*>(y_lo + orow * C + c0) = lo;
            }
        }
    }
    }
}

// Bulk-copy-staged variant for plain rows (no residual add): each warp keeps TWO rows in flight as 1-D cp.async.bulk copies into its own
// shared-memory slots (completion on an mbarrier), so the next row streams in while the current one is reduced, normalised and
// stored.  The register version above holds a row in 4 * MAXV registers per lane, which limits the SM to 32 warps and leaves
// their loads exposed: 2.6 TB/s at 32768 x 1280 from a cold L2 (tools/ln_micro.py); the staged rows cost no registers.
template <int MAXV>
__global__ void __launch_bounds__(256)
layernorm_bulk_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                      float* __restrict__ y_f32, __nv_bfloat16* __restrict__ y_hi, __nv_bfloat16* __restrict__ y_lo,
                      int64_t rows, int C, const int* __restrict__ omap, int y_fp16, uint8_t* __restrict__ y8) {
    extern __shared__ __align__(128) uint8_t ln_smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int nv = C >> 7;
    const uint32_t row_bytes = (uint32_t)C * 4u;
    float* slots = reinterpret_cast<float*>(ln_smem) + (size_t)warp * 2 * C;              // [2][C] per warp
    uint64_t* bars = reinterpret_cast<uint64_t*>(ln_smem + (size_t)8 * 2 * C * 4) + warp * 2;
    if (lane == 0) {
        ptx::mbar_init(&bars[0], 1);
        ptx::mbar_init(&bars[1], 1);
        ptx::fence_barrier_init();
    }
    __syncwarp();
    const int64_t wstride = ((int64_t)gridDim.x * blockDim.x) >> 5;
    int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    auto issue = [&](int64_t r, int st) {
        if (lane == 0) {
            ptx::fence_proxy_async_smem();                 // the slot's previous generic-proxy reads are ordered before the async write
            ptx::mbar_arrive_expect_tx(&bars[st], row_bytes);
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                             ptx::smem_u32(slots + (size_t)st * C)),
                         "l"(x + r * C), "r"(row_bytes), "r"(ptx::smem_u32(&bars[st]))
                         : "memory");
        }
    };
    if (row < rows) issue(row, 0);
    uint32_t ph[2] = {0u, 0u};
    for (int it = 0; row < rows; row += wstride, ++it) {
        const int st = it & 1;
        if (row + wstride < rows) issue(row + wstride, st ^ 1);
        ptx::mbar_wait(&bars[st], ph[st]);
        ph[st] ^= 1u;
        const float* xr = slots + (size_t)st * C;
        const int64_t orow = omap ? omap[row] : row;
        float4 v[MAXV];
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < MAXV; ++i) {
            if (i < nv) {
                v[i] = *reinterpret_cast<const float4*>(xr + (i * 32 + lane) * 4);
                s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
            }
        }
        __syncwarp();                                      // every lane has read the slot: it may be refilled two iterations from now
        const float mean = warp_sum(s) / (float)C;
        float q = 0.f;
#pragma unroll
        for (int i = 0; i < MAXV; ++i) {
            if (i < nv) {
                const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
                q += (a * a + b * b) + (c * c + d * d);
            }
        }
        const float rstd = rsqrtf(warp_sum(q) / (float)C + eps);
#pragma unroll
        for (int i = 0; i < MAXV; ++i) {
            if (i < nv) {
                const int c0 = (i * 32 + lane) * 4;
                const float4 g = *reinterpret_cast<const float4*>(gamma + c0);
                const float4 b = *reinterpret_cast<const float4*>(beta + c0);
                float4 o;
                o.x = (v[i].x - mean) * rstd * g.x + b.x;
                o.y = (v[i].y - mean) * rstd * g.y + b.y;
                o.z = (v[i].z - mean) * rstd * g.z + b.z;
                o.w = (v[i].w - mean) * rstd * g.w + b.w;
                if (y_f32) *reinterpret_cast<float4*>(y_f32 + orow * C + c0) = o;
                if (y_hi && y8) {
                    uint2 h16;
                    uint32_t a8, b8;
                    split4_f16_e4m3(o, h16, a8, b8);
                    *reinterpret_cast<uint2*>(y_hi + orow * C + c0) = h16;
                    uint8_t* o8 = y8 + orow * 2 * C + e4m3_slot0(c0);
                    *reinterpret_cast<uint32_t*>(o8) = a8;
                    *reinterpret_cast<uint32_t*>(o8 + 32) = b8;
                } else if (y_hi) {
                    uint2 hi, lo;
                    split2m(o.x, o.y, hi.x, lo.x, y_fp16);
                    split2m(o.z, o.w, hi.y, lo.y, y_fp16);
                    *reinterpret_cast<uint2*>(y_hi + orow * C + c0) = hi;
                    if (y_lo) *reinterpret_cast<uint2*>(y_lo + orow * C + c0) = lo;
                }
            }
        }
    }
}

// generic C: one block (128 threads) per row
__global__ void __launch_bounds__(128)
layernorm_generic_kernel(const float* __restrict__ x, const float* __restrict__ add,
                         const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                         float* __restrict__ sum_out, float* __restrict__ y_f32,
                         __nv_bfloat16* __restrict__ y_hi, __nv_bfloat16* __restrict__ y_lo, int64_t rows, int C,
                         const int* __restrict__ omap, int y_fp16, uint8_t* __restrict__ y8) {
    __shared__ float red[4];
    __shared__ float bc;
    const int64_t row = blockIdx.x;
    const int64_t orow = omap ? omap[row] : row;
    const float* xr = x + row * C;
    const float* ar = add ? add + row * C : nullptr;
    auto block_sum = [&](float v) {
        v = warp_sum(v);
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
        __syncthreads();
        if (threadIdx.x == 0) bc = red[0] + red[1] + red[2] + red[3];
        __syncthreads();
        const float r = bc;
        __syncthreads();
        return r;
    };
    float s = 0.f;
    for (int c = threadIdx.x; c < C; c += 128) {
        float v = xr[c] + (ar ? ar[c] : 0.f);
        if (ar && sum_out) sum_out[row * C + c] = v;
        s += v;
    }
    const float mean = block_sum(s) / (float)C;
    float q = 0.f;
    for (int c = threadIdx.x; c < C; c += 128) {
        const float v = xr[c] + (ar ? ar[c] : 0.f) - mean;
        q += v * v;
    }
    const float rstd = rsqrtf(block_sum(q) / (float)C + eps);
    for (int c = threadIdx.x; c < C; c += 128) {
        const float v = xr[c] + (ar ? ar[c] : 0.f);
        const float o = (v - mean) * rstd * gamma[c] + beta[c];
        if (y_f32) y_f32[orow * C + c] = o;
        if (y_hi && y_fp16) {
            const __half h = __float2half_rn(o);
            reinterpret_cast<__half*>(y_hi)[orow * C + c] = h;
            if (y8) {
                y8[orow * 2 * C + e4m3_slot0(c)] = (uint8_t)__nv_cvt_float_to_fp8(__half2float(h), __NV_SATFINITE, __NV_E4M3);
                y8[orow * 2 * C + e4m3_slot0(c) + 32] = (uint8_t)__nv_cvt_float_to_fp8((o - __half2float(h)) * 1024.f, __NV_SATFINITE, __NV_E4M3);
            }
        } else if (y_hi) {
            const __nv_bfloat16 h = __float2bfloat16_rn(o);
            y_hi[orow * C + c] = h;
            if (y_lo) y_lo[orow * C + c] = __float2bfloat16_rn(o - __bfloat162float(h));
        }
    }
}

// ---- GroupNorm on NHWC (rows = pixels, C channels), stats per (n, group) ---------------------
// pass 1: per-block partial sums -> double atomics into stats[n][g][2]
__global__ void __launch_bounds__(256)
groupnorm_stats_kernel(const float* __restrict__ x, double* __restrict__ stats, int HW, int C, int G,
                       int64_t x_bstride, int rows_per_block) {
    extern __shared__ float sm[];  // [2][G] partials
    const int n = blockIdx.y;
    const int cpg = C / G;
    for (int i = threadIdx.x; i < 2 * G; i += blockDim.x) sm[i] = 0.f;
    __syncthreads();
    const int r0 = blockIdx.x * rows_per_block;
    const int r1 = min(HW, r0 + rows_per_block);
    const float* xb = x + (int64_t)n * x_bstride;
    // thread handles a fixed channel (threadIdx.x % C) across rows when 256 % C == 0 or C % 256 == 0
    for (int c = threadIdx.x % C; c < C; c += (blockDim.x >= C ? C : blockDim.x)) {
        float s = 0.f, q = 0.f;
        const int rstep = blockDim.x >= C ? blockDim.x / C : 1;
        const int roff = blockDim.x >= C ? threadIdx.x / C : 0;
        for (int r = r0 + roff; r < r1; r += rstep) {
            const float v = xb[(int64_t)r * C + c];
            s += v;
            q += v * v;
        }
        atomicAdd(&sm[c / cpg], s);
        atomicAdd(&sm[G + c / cpg], q);
        if (blockDim.x >= C) break;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < G; i += blockDim.x) {
        atomicAdd(&stats[((int64_t)n * G + i) * 2], (double)sm[i]);
        atomicAdd(&stats[((int64_t)n * G + i) * 2 + 1], (double)sm[G + i]);
    }
}

__global__ void __launch_bounds__(256)
groupnorm_apply_kernel(const float* __restrict__ x, const double* __restrict__ stats,
                       const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                       const float* __restrict__ post_add, float* __restrict__ y_f32,
                       __nv_bfloat16* __restrict__ y_hi, __nv_bfloat16* __restrict__ y_lo, int HW, int C, int G,
                       int relu, int64_t x_bstride, int64_t y_bstride, int64_t add_bstride) {
    const int n = blockIdx.y;
    const int cpg = C / G;
    const int64_t total4 = (int64_t)HW * C / 4;
    const double cnt = (double)HW * cpg;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t e = i * 4;
        const int c = (int)(e % C);
        const int g = c / cpg;  // 4 consecutive channels share a group when cpg % 4 == 0
        const double mean_d = stats[((int64_t)n * G + g) * 2] / cnt;
        const double var_d = stats[((int64_t)n * G + g) * 2 + 1] / cnt - mean_d * mean_d;
        const float mean = (float)mean_d;
        const float rstd = (float)(1.0 / sqrt((var_d > 0 ? var_d : 0) + (double)eps));
        const float4 v = *reinterpret_cast<const float4*>(x + (int64_t)n * x_bstride + e);
        const float4 gm = *reinterpret_cast<const float4*>(gamma + c);
        const float4 bt = *reinterpret_cast<const float4*>(beta + c);
        float4 o;
        o.x = (v.x - mean) * rstd * gm.x + bt.x;
        o.y = (v.y - mean) * rstd * gm.y + bt.y;
        o.z = (v.z - mean) * rstd * gm.z + bt.z;
        o.w = (v.w - mean) * rstd * gm.w + bt.w;
        if (relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f); }
        if (post_add) {
            const float4 a = *reinterpret_cast<const float4*>(post_add + (int64_t)n * add_bstride + e);
            o.x += a.x; o.y += a.y; o.z += a.z; o.w += a.w;
        }
        if (y_f32) *reinterpret_cast<float4*>(y_f32 + (int64_t)n * y_bstride + e) = o;
        if (y_hi) {
            uint2 hi, lo;
            split2(o.x, o.y, hi.x, lo.x);
            split2(o.z, o.w, hi.y, lo.y);
            *reinterpret_cast<uint2*>(y_hi + (int64_t)n * y_bstride + e) = hi;
            if (y_lo) *reinterpret_cast<uint2*>(y_lo + (int64_t)n * y_bstride + e) = lo;
        }
    }
}

}  // namespace hipie

using namespace hipie;

// resident CTAs of layernorm_kernel<MAXV> on this device (register-limited: 4 per SM at MAXV = 10), queried once per instantiation
int g_ln_bulk = 1;            // hipie_set_option("ln_bulk", 0): register-resident rows only (A/B switch)
int g_ln_grid_cap = 1;        // hipie_set_option("ln_grid_cap", 0): one 8-row CTA per 8 rows as in round 1 (A/B switch)
template <int MAXV>
static int ln_resident_ctas() {
    if (!g_ln_grid_cap) return 0x7fffffff;
    static int n = 0;
    if (n == 0) {
        int per_sm = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, layernorm_kernel<MAXV>, 256, 0) != cudaSuccess || per_sm < 1) per_sm = 2;
        n = per_sm * num_sms();
    }
    return n;
}

static int layernorm_launch(const float* x, const float* add, const float* gamma, const float* beta, float eps,
                            float* sum_out, float* y_f32, void* y_hi, void* y_lo, int y_fp16, int64_t rows, int C,
                            const int32_t* out_row_map, void* stream, uint8_t* y8 = nullptr) {
    HIPIE_CHECK_ARG(x && gamma && beta, "hipie_layernorm: null input");
    HIPIE_CHECK_ARG(y_f32 || y_hi, "hipie_layernorm: no output requested");
    HIPIE_CHECK_ARG(rows >= 0 && C > 0, "hipie_layernorm: bad sizes");
    if (rows == 0) return HIPIE_OK;
    cudaStream_t st = (cudaStream_t)stream;
    __nv_bfloat16 *hi = (__nv_bfloat16*)y_hi, *lo = (__nv_bfloat16*)y_lo;
    if (g_ln_bulk && !add && C % 128 == 0 && C <= 128 * 10 && (reinterpret_cast<uintptr_t>(x) & 15) == 0 && rows >= 4096) {
        // rows staged by bulk copies: 2 slots of C floats per warp (80 KB per CTA at C = 1280)
        const int smem = 8 * 2 * C * 4 + 8 * 2 * 8;
        const int64_t want = (rows + 7) / 8;
        uint8_t* y8p = y8;
        if (C <= 128 * 2) {
            HIPIE_ENSURE_SMEM(layernorm_bulk_kernel<2>, smem);
            int per_sm = 0;
            if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, layernorm_bulk_kernel<2>, 256, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
            layernorm_bulk_kernel<2><<<(unsigned)std::min<int64_t>(want, (int64_t)per_sm * num_sms()), 256, smem, st>>>(x, gamma, beta, eps, y_f32, hi, lo, rows, C,
                                                                                                           out_row_map, y_fp16, y8p);
        } else if (C <= 128 * 6) {
            HIPIE_ENSURE_SMEM(layernorm_bulk_kernel<6>, smem);
            int per_sm = 0;
            if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, layernorm_bulk_kernel<6>, 256, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
            layernorm_bulk_kernel<6><<<(unsigned)std::min<int64_t>(want, (int64_t)per_sm * num_sms()), 256, smem, st>>>(x, gamma, beta, eps, y_f32, hi, lo, rows, C,
                                                                                                           out_row_map, y_fp16, y8p);
        } else {
            HIPIE_ENSURE_SMEM(layernorm_bulk_kernel<10>, smem);
            int per_sm = 0;
            if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, layernorm_bulk_kernel<10>, 256, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
            layernorm_bulk_kernel<10><<<(unsigned)std::min<int64_t>(want, (int64_t)per_sm * num_sms()), 256, smem, st>>>(x, gamma, beta, eps, y_f32, hi, lo, rows, C,
                                                                                                            out_row_map, y_fp16, y8p);
        }
    } else if (C % 128 == 0 && C <= 128 * 16) {
        const int64_t want = (rows + 7) / 8;
        int64_t blocks;
        if (C <= 128 * 2)
            layernorm_kernel<2><<<(unsigned)(blocks = std::min<int64_t>(want, ln_resident_ctas<2>())), 256, 0, st>>>(x, add, gamma, beta, eps, sum_out, y_f32, hi, lo, rows, C, out_row_map, y_fp16, y8);
        else if (C <= 128 * 6)
            layernorm_kernel<6><<<(unsigned)(blocks = std::min<int64_t>(want, ln_resident_ctas<6>())), 256, 0, st>>>(x, add, gamma, beta, eps, sum_out, y_f32, hi, lo, rows, C, out_row_map, y_fp16, y8);
        else if (C <= 128 * 10)
            layernorm_kernel<10><<<(unsigned)(blocks = std::min<int64_t>(want, ln_resident_ctas<10>())), 256, 0, st>>>(x, add, gamma, beta, eps, sum_out, y_f32, hi, lo, rows, C, out_row_map, y_fp16, y8);
        else
            layernorm_kernel<16><<<(unsigned)(blocks = std::min<int64_t>(want, ln_resident_ctas<16>())), 256, 0, st>>>(x, add, gamma, beta, eps, sum_out, y_f32, hi, lo, rows, C, out_row_map, y_fp16, y8);
    } else {
        layernorm_generic_kernel<<<(unsigned)rows, 128, 0, st>>>(x, add, gamma, beta, eps, sum_out, y_f32, hi, lo, rows, C, out_row_map, y_fp16, y8);
    }
    HIPIE_CHECK_LAUNCH();
    return HIPIE_OK;
}

extern "C" int hipie_layernorm(const float* x, const float* add, const float* gamma, const float* beta, float eps,
                               float* sum_out, float* y_f32, void* y_hi, void* y_lo, int64_t rows, int C,
                               const int32_t* out_row_map, void* stream) {
    return layernorm_launch(x, add, gamma, beta, eps, sum_out, y_f32, y_hi, y_lo, 0, rows, C, out_row_map, stream);
}

extern "C" int hipie_layernorm_f16(const float* x, const float* add, const float* gamma, const float* beta, float eps,
                                   float* sum_out, float* y_f32, void* y_f16, void* y_e4m3, int64_t rows, int C,
                                   const int32_t* out_row_map, void* stream) {
    HIPIE_CHECK_ARG(y_f16 != nullptr, "hipie_layernorm_f16: y_f16 required");
    HIPIE_CHECK_ARG(!y_e4m3 || C % 32 == 0, "hipie_layernorm_f16: the e4m3 planes need C %% 32 == 0");
    return layernorm_launch(x, add, gamma, beta, eps, sum_out, y_f32, y_f16, nullptr, 1, rows, C, out_row_map, stream, (uint8_t*)y_e4m3);
}

extern "C" int hipie_groupnorm_nhwc(const float* x, const float* gamma, const float* beta, float eps,
                                    const float* post_add, float* y_f32, void* y_hi, void* y_lo, double* stats_ws,
                                    int N, int HW, int C, int G, int relu, int64_t x_bstride, int64_t y_bstride,
                                    int64_t add_bstride, void* stream) {
    HIPIE_CHECK_ARG(x && gamma && beta && stats_ws, "hipie_groupnorm_nhwc: null input");
    HIPIE_CHECK_ARG(y_f32 || y_hi, "hipie_groupnorm_nhwc: no output requested");
    HIPIE_CHECK_ARG(N > 0 && HW > 0 && C > 0 && G > 0 && C % G == 0 && (C / G) % 4 == 0 && C <= 1024,
                    "hipie_groupnorm_nhwc: bad sizes N=%d HW=%d C=%d G=%d", N, HW, C, G);
    HIPIE_CHECK_ARG(256 % C == 0 || C % 256 == 0, "hipie_groupnorm_nhwc: C must divide or be a multiple of 256");
    cudaStream_t st = (cudaStream_t)stream;
    HIPIE_CHECK_CUDA(cudaMemsetAsync(stats_ws, 0, sizeof(double) * 2 * N * G, st));
    const int rows_per_block = 64;
    dim3 g1((HW + rows_per_block - 1) / rows_per_block, N);
    groupnorm_stats_kernel<<<g1, 256, 2 * G * sizeof(float), st>>>(x, stats_ws, HW, C, G, x_bstride, rows_per_block);
    HIPIE_CHECK_LAUNCH();
    const int64_t total4 = (int64_t)HW * C / 4;
    int bx = (int)((total4 + 255) / 256);
    if (bx > num_sms() * 8) bx = num_sms() * 8;
    dim3 g2(bx, N);
    groupnorm_apply_kernel<<<g2, 256, 0, st>>>(x, stats_ws, gamma, beta, eps, post_add, y_f32, (__nv_bfloat16*)y_hi,
                                               (__nv_bfloat16*)y_lo, HW, C, G, relu, x_bstride, y_bstride, add_bstride);
    HIPIE_CHECK_LAUNCH();
    return HIPIE_OK;
}
