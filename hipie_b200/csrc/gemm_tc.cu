// Persistent, warp-specialised wgmma GEMM for sm_90a (H100):
//   C[b] = epilogue( alpha * A[b] . W[b]^T )      A: (M,K) bf16 K-major,  W: (N,K) bf16 K-major
//
// This one kernel carries every dense contraction of the hot path: the ViT-H qkv / proj / fc1 / fc2 linears (reference
// hipie/backbone/vit.py:67-83,212-230), the DETR / MaskDINO / BERT linears, convolutions lowered to GEMM, and the MaskDINO
// mask-embed contraction einsum("bqc,bchw->bqhw") (.../maskdino/transformer_decoder/maskdino_decoder.py:520-529) with the
// sigmoid-threshold fused as a bit-packed output.
//
// Structure (one CTA per SM, 384 threads, 128 x BN tiles, BN = 64, 128 or 256):
//   warpgroup 0     TMA producer (one thread): cp.async.bulk.tensor tiles of A / W into a 3-4 stage 128B/64B-swizzled
//                   shared-memory ring, completion on mbarriers (expect_tx)
//   warpgroups 1-2  consumers, 64 tile rows each: wgmma (m64 x BN x 16, both operands from shared memory) into fp32 register
//                   accumulators, one k-block in flight, then the fused epilogue: bias / activation / layer-scale / residual,
//                   fp32 + bf16-split / fp16 / fp16 + e4m3 + bit-packed outputs, row-major through TMA stores where possible.
//   BN = 64 / 128:  the accumulator is staged row-major in shared memory and each warp runs the epilogue on 32 rows x BN/2
//                   columns; this path also writes the transposed outputs (the attention's V^T) and the bit-packed mask.
//   BN = 256:       the ViT-H linears (prec 4 and 6, row-major).  A quarter fewer operand bytes per flop than 128 x 128, so more of the
//                   L2 -> shared-memory feed turns into tensor work.  128 accumulators per consumer thread (setmaxnreg: 40
//                   producer + 2 x 232 consumer registers); the staged tile would take 132 KB, so each warp runs the epilogue
//                   straight from its 16 fragment rows (epilogue_frag), and a 4-stage ring fits (48 KB stages for prec 6).
//
// Precision: operands are bf16 "split" planes.  prec==1 uses hi only; prec==3 computes
// Ahi.Whi + Ahi.Wlo + Alo.Whi in the same fp32 accumulator (error ~2^-16 relative, i.e.
// fp32-class results from the bf16 tensor pipe), loading 4 tiles per 3 MMAs per k-block.
// prec==4 is the two-pass fp16 mode of the precision map (DESIGN.md 3): A is ONE IEEE fp16 plane (an activation that is
// rounded to fp16 downstream anyway: the LayerNorm output feeding qkv), W is fp16 hi + lo, A.Whi + A.Wlo -- the weight is exact
// to ~2^-22, the only rounding is the 2^-12 of the activation plane; 3 tiles per 2 MMAs per k-block.
// prec==6 is the fp16 + e4m3 split (the large ViT linears): with A = Ah + Al, W = Wh + Wl (fp16 hi, exact remainders)
//     A.W = Ah.Wh  +  2^-14 * ( e4m3(Ah) . e4m3(2^14 Wl)  +  e4m3(2^10 Al) . e4m3(2^4 Wh) )  +  O(2^-16 |A||W|)
// The cross terms are 2^-11 of the product, so the 2^-4 relative rounding of their e4m3 factors lands at 2^-15..2^-16 -- the
// class of the bf16x3 scheme (tools/prec_map_emulate.py: mask logits unchanged at 1.4e-4) -- and both of them are ONE fp8
// contraction over 2K: operand planes A8 = [e4m3(Ah) | e4m3(2^10 Al)] (M x 2K) and W8 = [e4m3(2^14 Wl) | e4m3(2^4 Wh)]
// (N x 2K), the two slots interleaved in 32-column groups (common.cuh: e4m3_slot0) so that producers write 64-byte row segments.
// Per tile the consumers first sweep the fp8 planes (m64nNk32 e4m3 wgmma: twice the rate of the 16-bit kinds), accumulating
// 2^14 x the cross terms, scale the accumulator by 2^-14 in registers, then sweep the fp16 planes.  Two pass-equivalents
// instead of three, same operand bytes.
#include "common.cuh"
#include "ptx.cuh"
#include "wgmma.cuh"
#include <mutex>
#include <type_traits>
#include <unordered_map>
#include <string.h>

namespace hipie {
using namespace ptx;

constexpr int GEMM_BM = 128;
constexpr int GEMM_CONSUMERS = 2;                            // warpgroups, 64 accumulator rows each
constexpr int GEMM_EPI_WARPS = 4 * GEMM_CONSUMERS;
constexpr int GEMM_THREADS = 128 + 128 * GEMM_CONSUMERS;     // producer warpgroup (one TMA thread) + the consumer warpgroups
// setmaxnreg split of the 168 registers per thread of the 128 x 256 tiles (128 fp32 accumulators per consumer thread): 40 + 2 x 232
constexpr int GEMM_PRODUCER_REGS = 40, GEMM_CONSUMER_REGS = 232;
constexpr int EPI_LD = 16;  // row length (floats) of the epilogue transpose buffer; 16-byte groups are XOR-swizzled by row
constexpr int EPI_WARP_BYTES = 4096;   // per epilogue warp: one 32 x 32 fp32 TMA-store box (or a 32 x 32 bf16 hi box + lo box)

struct GemmParams {
    const float* bias;
    const float* colscale;
    const float* residual;
    int64_t ldr, r_bstride;
    float* c_f32;
    __nv_bfloat16* c_hi;
    __nv_bfloat16* c_lo;
    int64_t ldc, c_bstride;
    uint32_t* c_bits;
    float bits_threshold;
    int M, N, K, batch;
    int act;
    float alpha;
    int transposed;  // 1: C stored as [N, ldc] (column-major output), lanes = rows; 2 / 3: the vectorised fp16-plane variant (8 / 4 rows per store)
    int tiles_m, tiles_n;
    int f16_ops;     // operands are IEEE fp16 planes: fp16 wgmma instead of bf16
    int relu_post;   // ReLU after the residual add
    int c_fp16;      // c_hi is one IEEE fp16 plane instead of bf16 hi/lo
    int c_e4m3;      // ... plus the e4m3 planes [e4m3(h) | e4m3(2^10 (x - h))] of the result (M x 2N, TMA-store path, map tm_c_lo)
    int tma_out;     // row-major outputs leave through TMA stores (32 x 32 boxes staged in swizzled shared memory)
    int m_fastest;   // tile order: 1 = the few M tiles of one N tile run back to back (concurrently on neighbouring SMs), so the
                     // big streamed W operand is fetched from HBM once and re-read from L2 (short, wide problems)
    const int* row_map;
    int t_row_group, t_row_pad;   // transposed epilogue: row r -> r + (r / group) * pad (0 = off)
};

template <int PREC, int BN>
struct GemmCfg {
    static constexpr bool P4 = PREC == 4;
    static constexpr bool P6 = PREC == 6;                    // fp16 hi.hi sweep + e4m3 sweep for the two cross terms (see the header comment)
    static constexpr bool WIDE = BN == 256;                  // prec 4 / 6 only: epilogue from the register fragment, no staged tile
    static constexpr int BK = (PREC == 3 || P4) ? 32 : 64;   // elements per k-block of the 16-bit operands; BK*2 bytes == swizzle span
    static constexpr int BK8 = 128;                          // elements (= bytes) per k-block of the e4m3 sweep
    static constexpr int SWZ = BK * 2;
    static constexpr int A_TILE = GEMM_BM * BK * 2;          // bytes
    static constexpr int W_TILE = BN * BK * 2;
    static constexpr int A_PLANES = PREC == 3 ? 2 : 1, W_PLANES = (PREC == 3 || P4) ? 2 : 1;     // prec 6: one plane per sweep, same tile bytes
    static constexpr int STAGE = A_PLANES * A_TILE + W_PLANES * W_TILE;     // layout: A_hi | W_hi | (A_lo) | W_lo
    static constexpr int ACC_LD = BN + 4;                    // fp32 accumulator tile staged for the epilogue: padded rows, lane = row reads
    static constexpr int ACC_BYTES = WIDE ? 0 : GEMM_BM * ACC_LD * 4;  //   are conflict-free
    static constexpr int EPI_BYTES = GEMM_EPI_WARPS * EPI_WARP_BYTES;
    static constexpr int SMEM_BUDGET = 232448 - 1024 - 256 - EPI_BYTES - ACC_BYTES;      // 227 KB per CTA
    static constexpr int MAX_STAGES = 4;
    static constexpr int STAGES = SMEM_BUDGET / STAGE < MAX_STAGES ? SMEM_BUDGET / STAGE : MAX_STAGES;
    static_assert(STAGES >= 3, "pipeline too shallow");
    static_assert(!WIDE || (STAGES == 4 && (P4 || P6)), "the 128 x 256 tiles run prec 4 / 6 on a 4-stage ring");
    static constexpr int SMEM = STAGES * STAGE + ACC_BYTES + EPI_BYTES + 256 + 1024;
};

// NV fp32 values of one accumulator row (lane = row of the staged tile)
template <int NV>
__device__ __forceinline__ void acc_ld(const float* row, uint32_t (&v)[NV]) {
#pragma unroll
    for (int i = 0; i < NV; i += 4) {
        const uint4 q = *reinterpret_cast<const uint4*>(row + i);
        v[i] = q.x; v[i + 1] = q.y; v[i + 2] = q.z; v[i + 3] = q.w;
    }
}

__device__ __forceinline__ float act_apply(float v, int act) {
    if (act == HIPIE_ACT_RELU) return fmaxf(v, 0.f);
    if (act == HIPIE_ACT_GELU) return 0.5f * v * (1.f + erff(v * 0.70710678118654752440f));
    if (act == HIPIE_ACT_SIGMOID) return 1.f / (1.f + expf(-v));
    if (act == HIPIE_ACT_QUICK_GELU) return v / (1.f + expf(-1.702f * v));
    return v;
}

// QuickGELU (x * sigmoid(1.702 x): OpenAI CLIP's activation, open_clip model.py QuickGELU) shares the SIGMOID instantiation of
// the epilogues -- one uniform flag instead of a fourth copy of every epilogue
template <int ACT>
__device__ __forceinline__ float act_apply_t(float v, bool quick) {
    if (ACT == HIPIE_ACT_RELU) return fmaxf(v, 0.f);
    if (ACT == HIPIE_ACT_GELU) return 0.5f * v * (1.f + erff(v * 0.70710678118654752440f));
    if (ACT == HIPIE_ACT_SIGMOID) return quick ? v / (1.f + expf(-1.702f * v)) : 1.f / (1.f + expf(-v));
    return v;
}

// Row-major bit-packed output: bits[b][row][col / 32], bit (col % 32) = value > threshold.  The four lanes that hold the 16
// columns [col16, col16 + 16) of one row (4 each) combine their nibbles and lane 0 of the group stores one 16-bit half word.
__device__ __forceinline__ void row_bits16(const GemmParams& p, const float4& x, int b, int row, int col16, int lane) {
    uint32_t v = (x.x > p.bits_threshold ? 1u : 0u) | (x.y > p.bits_threshold ? 2u : 0u) | (x.z > p.bits_threshold ? 4u : 0u) |
                 (x.w > p.bits_threshold ? 8u : 0u);
    v <<= 4 * (lane & 3);
    const uint32_t gmask = 0xfu << (lane & ~3);
    v |= __shfl_xor_sync(gmask, v, 1);
    v |= __shfl_xor_sync(gmask, v, 2);
    if ((lane & 3) == 0) {
        const int64_t words_per_row = (p.N + 31) / 32;
        uint16_t* dst = reinterpret_cast<uint16_t*>(p.c_bits + ((int64_t)b * p.M + row) * words_per_row);
        dst[col16 >> 4] = (uint16_t)v;
    }
}

__device__ __forceinline__ void sts128(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
    asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ float4 lds128(uint32_t addr) {
    float4 r;
    asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "r"(addr) : "memory");
    return r;
}

// Interior-tile row epilogue: all 32 rows and all columns of the warp's slice are in range, rows are 16-byte aligned and
// not remapped.  No per-element predicates, 32-bit offsets from one tile base, the next chunk's accumulator load is in flight
// while the current chunk is converted and stored.
template <int ACT>
__device__ __forceinline__ void epilogue_rows_fast(const GemmParams& p, const float* arow, uint32_t es, int b, int m0, int n0,
                                                   int col_begin, int col_end, int lane) {
    const int rsub = lane >> 2, c4 = (lane & 3) * 4;
    const int64_t tile_c = (int64_t)b * p.c_bstride + (int64_t)m0 * p.ldc + n0 + c4;
    const float* res_t = p.residual ? p.residual + (int64_t)b * p.r_bstride + (int64_t)m0 * p.ldr + n0 + c4 : nullptr;
    float* cf_t = p.c_f32 ? p.c_f32 + tile_c : nullptr;
    __nv_bfloat16* chi_t = p.c_hi ? p.c_hi + tile_c : nullptr;
    __nv_bfloat16* clo_t = p.c_lo ? p.c_lo + tile_c : nullptr;
    const float* bias_t = p.bias ? p.bias + n0 + c4 : nullptr;
    const float* cs_t = p.colscale ? p.colscale + n0 + c4 : nullptr;
    const int ldc = (int)p.ldc, ldr = (int)p.ldr;
    const float alpha = p.alpha;
    const uint32_t wr = es + lane * (EPI_LD * 4);
    const uint32_t wsw = (lane >> 1) & 3;
    uint32_t v[16];
    acc_ld(arow + col_begin, v);
#pragma unroll 1
    for (int cb = col_begin; cb < col_end; cb += 16) {
#pragma unroll
        for (int j = 0; j < 4; ++j) sts128(wr + ((j ^ wsw) << 4), v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
        __syncwarp();
        if (cb + 16 < col_end) acc_ld(arow + cb + 16, v);
        float4 bias = make_float4(0.f, 0.f, 0.f, 0.f), cs = make_float4(1.f, 1.f, 1.f, 1.f);
        if (bias_t) bias = *reinterpret_cast<const float4*>(bias_t + cb);
        if (cs_t) cs = *reinterpret_cast<const float4*>(cs_t + cb);
#pragma unroll
        for (int it = 0; it < 4; ++it) {
            const int rr = it * 8 + rsub;
            float4 x = lds128(es + rr * (EPI_LD * 4) + (((lane & 3) ^ ((rr >> 1) & 3)) << 4));
            x.x = act_apply_t<ACT>(fmaf(x.x, alpha, bias.x), p.act == HIPIE_ACT_QUICK_GELU);
            x.y = act_apply_t<ACT>(fmaf(x.y, alpha, bias.y), p.act == HIPIE_ACT_QUICK_GELU);
            x.z = act_apply_t<ACT>(fmaf(x.z, alpha, bias.z), p.act == HIPIE_ACT_QUICK_GELU);
            x.w = act_apply_t<ACT>(fmaf(x.w, alpha, bias.w), p.act == HIPIE_ACT_QUICK_GELU);
            if (cs_t) { x.x *= cs.x; x.y *= cs.y; x.z *= cs.z; x.w *= cs.w; }
            if (res_t) {
                const float4 rv = *reinterpret_cast<const float4*>(res_t + rr * ldr + cb);
                x.x += rv.x; x.y += rv.y; x.z += rv.z; x.w += rv.w;
            }
            if (p.relu_post) { x.x = fmaxf(x.x, 0.f); x.y = fmaxf(x.y, 0.f); x.z = fmaxf(x.z, 0.f); x.w = fmaxf(x.w, 0.f); }
            const int off = rr * ldc + cb;
            if (p.c_bits) row_bits16(p, x, b, m0 + rr, n0 + cb, lane);
            if (cf_t) *reinterpret_cast<float4*>(cf_t + off) = x;
            if (chi_t) {
                uint2 hi, lo;
                split2m(x.x, x.y, hi.x, lo.x, p.c_fp16);
                split2m(x.z, x.w, hi.y, lo.y, p.c_fp16);
                *reinterpret_cast<uint2*>(chi_t + off) = hi;
                if (clo_t) *reinterpret_cast<uint2*>(clo_t + off) = lo;
            }
        }
        __syncwarp();
    }
}

// Row-major epilogue for one warp: `nch` chunks of 32 columns starting at chunk c0.  The accumulator rows
// (one per lane) are transposed through padded smem; afterwards lanes 0-7 cover one row with float4s, so a
// warp stores four fully coalesced 128-byte row segments per instruction.
template <int ACT>
__device__ __forceinline__ void epilogue_rows(const GemmParams& p, const float* arow, float* my_epi, int b, int m0,
                                              int n0, int col_begin, int col_end, int lane) {
    const float* res_b = p.residual ? p.residual + (int64_t)b * p.r_bstride : nullptr;
    float* cf_b = p.c_f32 ? p.c_f32 + (int64_t)b * p.c_bstride : nullptr;
    __nv_bfloat16* chi_b = p.c_hi ? p.c_hi + (int64_t)b * p.c_bstride : nullptr;
    __nv_bfloat16* clo_b = p.c_lo ? p.c_lo + (int64_t)b * p.c_bstride : nullptr;
    const int rsub = lane >> 2, c4 = (lane & 3) * 4;   // 8 rows x 16 columns per warp instruction
    const bool vec_ok = ((p.ldc & 3) == 0) && (!res_b || (p.ldr & 3) == 0);
    const int rmax = min(32, p.M - m0);
    if (vec_ok && !p.row_map && rmax == 32 && n0 + col_end <= p.N && 32 * p.ldc < (1ll << 30) && ((n0 & 3) == 0)) {
        epilogue_rows_fast<ACT>(p, arow, smem_u32(my_epi), b, m0, n0, col_begin, col_end, lane);
        return;
    }
#pragma unroll 1
    for (int cb = col_begin; cb < col_end; cb += 16) {
        const int nbase = n0 + cb;
        if (nbase >= p.N) break;  // warp-uniform
        uint32_t v[16];
        acc_ld(arow + cb, v);
#pragma unroll
        for (int j = 0; j < 16; j += 4)     // 16-byte group g of row r lives at group g ^ ((r >> 1) & 3): conflict-free both ways
            *reinterpret_cast<uint4*>(my_epi + lane * EPI_LD + (((j >> 2) ^ ((lane >> 1) & 3)) << 2)) =
                make_uint4(v[j], v[j + 1], v[j + 2], v[j + 3]);
        __syncwarp();
        const int col = nbase + c4;
        float4 bias = make_float4(0.f, 0.f, 0.f, 0.f), cs = make_float4(1.f, 1.f, 1.f, 1.f);
        const bool full4 = col + 3 < p.N;
        if (p.bias) {
            if (full4) bias = *reinterpret_cast<const float4*>(p.bias + col);
            else {
                if (col < p.N) bias.x = p.bias[col];
                if (col + 1 < p.N) bias.y = p.bias[col + 1];
                if (col + 2 < p.N) bias.z = p.bias[col + 2];
            }
        }
        if (p.colscale) {
            if (full4) cs = *reinterpret_cast<const float4*>(p.colscale + col);
            else {
                if (col < p.N) cs.x = p.colscale[col];
                if (col + 1 < p.N) cs.y = p.colscale[col + 1];
                if (col + 2 < p.N) cs.z = p.colscale[col + 2];
            }
        }
#pragma unroll
        for (int it = 0; it < 4; ++it) {
            const int rr = it * 8 + rsub;
            if (rr >= rmax || col >= p.N) continue;
            float4 x = *reinterpret_cast<const float4*>(my_epi + rr * EPI_LD + (((lane & 3) ^ ((rr >> 1) & 3)) << 2));
            x.x = act_apply_t<ACT>(x.x * p.alpha + bias.x, p.act == HIPIE_ACT_QUICK_GELU) * cs.x;
            x.y = act_apply_t<ACT>(x.y * p.alpha + bias.y, p.act == HIPIE_ACT_QUICK_GELU) * cs.y;
            x.z = act_apply_t<ACT>(x.z * p.alpha + bias.z, p.act == HIPIE_ACT_QUICK_GELU) * cs.z;
            x.w = act_apply_t<ACT>(x.w * p.alpha + bias.w, p.act == HIPIE_ACT_QUICK_GELU) * cs.w;
            int64_t row = m0 + rr;
            if (p.row_map) {
                row = p.row_map[(int64_t)b * p.M + row];
                if (row < 0) continue;
            }
            const int64_t off = row * p.ldc + col;
            if (full4 && vec_ok) {
                if (res_b) {
                    const float4 rv = *reinterpret_cast<const float4*>(res_b + row * p.ldr + col);
                    x.x += rv.x; x.y += rv.y; x.z += rv.z; x.w += rv.w;
                }
                if (p.relu_post) { x.x = fmaxf(x.x, 0.f); x.y = fmaxf(x.y, 0.f); x.z = fmaxf(x.z, 0.f); x.w = fmaxf(x.w, 0.f); }
                if (p.c_bits) row_bits16(p, x, b, (int)row, nbase, lane);
                if (cf_b) *reinterpret_cast<float4*>(cf_b + off) = x;
                if (chi_b) {
                    uint2 hi, lo;
                    split2m(x.x, x.y, hi.x, lo.x, p.c_fp16);
                    split2m(x.z, x.w, hi.y, lo.y, p.c_fp16);
                    *reinterpret_cast<uint2*>(chi_b + off) = hi;
                    if (clo_b) *reinterpret_cast<uint2*>(clo_b + off) = lo;
                }
            } else {
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    if (col + e < p.N) {
                        float xv = e == 0 ? x.x : (e == 1 ? x.y : (e == 2 ? x.z : x.w));
                        if (res_b) xv += res_b[row * p.ldr + col + e];
                        if (p.relu_post) xv = fmaxf(xv, 0.f);
                        if (cf_b) cf_b[off + e] = xv;
                        if (chi_b) {
                            if (p.c_fp16) {
                                reinterpret_cast<__half*>(chi_b)[off + e] = __float2half_rn(xv);
                            } else {
                                const __nv_bfloat16 h = __float2bfloat16_rn(xv);
                                chi_b[off + e] = h;
                                if (clo_b) clo_b[off + e] = __float2bfloat16_rn(xv - __bfloat162float(h));
                            }
                        }
                    }
                }
            }
        }
        __syncwarp();
    }
}

__device__ __forceinline__ float4 load4_guard(const float* p, int col, int N, float fill) {
    if (col + 3 < N) return *reinterpret_cast<const float4*>(p + col);
    float4 r = make_float4(fill, fill, fill, fill);
    if (col < N) r.x = p[col];
    if (col + 1 < N) r.y = p[col + 1];
    if (col + 2 < N) r.z = p[col + 2];
    return r;
}

// Row-major epilogue through TMA stores.  The warp reads 32 accumulator columns per step (lane = row), applies the fused
// bias / activation / layer-scale in that layout, writes the 32 x 32 box into its private staging buffer in the tensor map's
// swizzled layout (128 B rows for fp32, 64 B rows per bf16 plane: conflict-free 16-byte stores) and one lane hands the box to
// the TMA unit: full-line global writes that do not occupy the LSU, clipped at the matrix edges by the hardware.  The bit-packed
// (x > threshold) output falls out of the layout for free: a lane's 32 columns are one 32-bit word of its row.
template <int ACT>
__device__ __forceinline__ void epilogue_rows_tma(const GemmParams& p, const CUtensorMap* tm_f32, const CUtensorMap* tm_hi,
                                                  const CUtensorMap* tm_lo, const float* arow, uint32_t sbuf, int b, int m0, int n0,
                                                  int col_begin, int col_end, int lane) {
    if (m0 >= p.M) return;          // warp-uniform: this 32-row group lies below the matrix
    const float alpha = p.alpha;
    const int row = m0 + lane;
    const int npass = (p.c_f32 ? 1 : 0) + (p.c_hi ? 1 : 0);
#pragma unroll 1
    for (int cb = col_begin; cb < col_end; cb += 32) {
        const int nbase = n0 + cb;
        if (nbase >= p.N) break;  // warp-uniform
        uint32_t v[32];
        acc_ld(arow + cb, v);
#pragma unroll 1
        for (int pass = 0; pass < npass; ++pass) {
            const bool planes = p.c_hi && (pass == npass - 1) && !(p.c_f32 && pass == 0);
            // the previous box must have been read out of the staging buffer before it is overwritten
            if (lane == 0) bulk_wait_read0();
            __syncwarp();
            uint32_t word = 0;
            uint32_t h8[8], l8[8];
#pragma unroll
            for (int g = 0; g < 8; ++g) {
                const int col = nbase + 4 * g;
                float4 x = make_float4(__uint_as_float(v[4 * g]), __uint_as_float(v[4 * g + 1]), __uint_as_float(v[4 * g + 2]),
                                       __uint_as_float(v[4 * g + 3]));
                float4 bias = make_float4(0.f, 0.f, 0.f, 0.f);
                if (p.bias) bias = load4_guard(p.bias, col, p.N, 0.f);
                x.x = act_apply_t<ACT>(fmaf(x.x, alpha, bias.x), p.act == HIPIE_ACT_QUICK_GELU);
                x.y = act_apply_t<ACT>(fmaf(x.y, alpha, bias.y), p.act == HIPIE_ACT_QUICK_GELU);
                x.z = act_apply_t<ACT>(fmaf(x.z, alpha, bias.z), p.act == HIPIE_ACT_QUICK_GELU);
                x.w = act_apply_t<ACT>(fmaf(x.w, alpha, bias.w), p.act == HIPIE_ACT_QUICK_GELU);
                if (p.colscale) {
                    const float4 cs = load4_guard(p.colscale, col, p.N, 1.f);
                    x.x *= cs.x; x.y *= cs.y; x.z *= cs.z; x.w *= cs.w;
                }
                if (p.c_bits && pass == 0) {
                    word |= ((x.x > p.bits_threshold && col < p.N) ? 1u : 0u) << (4 * g);
                    word |= ((x.y > p.bits_threshold && col + 1 < p.N) ? 1u : 0u) << (4 * g + 1);
                    word |= ((x.z > p.bits_threshold && col + 2 < p.N) ? 1u : 0u) << (4 * g + 2);
                    word |= ((x.w > p.bits_threshold && col + 3 < p.N) ? 1u : 0u) << (4 * g + 3);
                }
                if (!planes) {
                    // fp32 box: 128-byte rows, 16-byte group g of row r at g ^ (r & 7)  (CU_TENSOR_MAP_SWIZZLE_128B)
                    sts128(sbuf + lane * 128 + ((g ^ (lane & 7)) << 4), __float_as_uint(x.x), __float_as_uint(x.y), __float_as_uint(x.z),
                           __float_as_uint(x.w));
                } else if (p.c_e4m3) {
                    // fp16 box as below + the two e4m3 boxes (32-byte rows, unswizzled) collected in registers
                    uint2 hi;
                    split4_f16_e4m3(x, hi, h8[g], l8[g]);
                    const uint32_t off = lane * 64 + (((g >> 1) ^ ((lane >> 1) & 3)) << 4) + ((g & 1) << 3);
                    asm volatile("st.shared.v2.b32 [%0], {%1,%2};" ::"r"(sbuf + off), "r"(hi.x), "r"(hi.y) : "memory");
                } else {
                    // bf16 boxes: 64-byte rows, 16-byte group c of row r at c ^ ((r >> 1) & 3)  (CU_TENSOR_MAP_SWIZZLE_64B)
                    uint2 hi, lo;
                    split2m(x.x, x.y, hi.x, lo.x, p.c_fp16);
                    split2m(x.z, x.w, hi.y, lo.y, p.c_fp16);
                    const uint32_t off = lane * 64 + (((g >> 1) ^ ((lane >> 1) & 3)) << 4) + ((g & 1) << 3);
                    asm volatile("st.shared.v2.b32 [%0], {%1,%2};" ::"r"(sbuf + off), "r"(hi.x), "r"(hi.y) : "memory");
                    if (p.c_lo) asm volatile("st.shared.v2.b32 [%0], {%1,%2};" ::"r"(sbuf + 2048 + off), "r"(lo.x), "r"(lo.y) : "memory");
                }
            }
            if (planes && p.c_e4m3) {
                // ONE e4m3 box: 64-byte rows = [slot 0: 32 bytes | slot 1: 32 bytes] of this 32-column chunk (the planes interleave the slots in
                // 32-column groups, common.cuh), 16-byte group c of row r at c ^ ((r >> 1) & 3)  (CU_TENSOR_MAP_SWIZZLE_64B)
                const uint32_t rb = sbuf + 2048 + lane * 64, sw = (lane >> 1) & 3;
                sts128(rb + ((0 ^ sw) << 4), h8[0], h8[1], h8[2], h8[3]);
                sts128(rb + ((1 ^ sw) << 4), h8[4], h8[5], h8[6], h8[7]);
                sts128(rb + ((2 ^ sw) << 4), l8[0], l8[1], l8[2], l8[3]);
                sts128(rb + ((3 ^ sw) << 4), l8[4], l8[5], l8[6], l8[7]);
            }
            fence_proxy_async_smem();      // generic-proxy writes -> visible to the TMA (async proxy)
            __syncwarp();
            if (lane == 0) {
                if (!planes) {
                    tma_store_3d(tm_f32, sbuf, nbase, m0, b);
                } else {
                    tma_store_3d(tm_hi, sbuf, nbase, m0, b);
                    if (p.c_e4m3) tma_store_3d(tm_lo, sbuf + 2048, 2 * nbase, m0, b);      // both slots of columns [nbase, nbase + 32): bytes [2 nbase, +64)
                    else if (p.c_lo) tma_store_3d(tm_lo, sbuf + 2048, nbase, m0, b);
                }
                bulk_commit();
            }
            if (p.c_bits && pass == 0 && row < p.M) {
                const int64_t words_per_row = (p.N + 31) / 32;
                p.c_bits[((int64_t)b * p.M + row) * words_per_row + (nbase >> 5)] = word;
            }
        }
    }
}

// Transposed fp16-plane epilogue (the V^T operand of the attention: C^T stored [col * ldc + row], one IEEE fp16 plane, bias only).
// A lane owns ONE row of the accumulator, so the scalar path below stores 2 bytes per lane and instruction (64-byte segments, 32
// store instructions per 32-column chunk: the V^T GEMM took the same 0.21 ms in one, two or three MMA passes).  Here the warp's
// 32 x 32 chunk goes through its shared-memory staging buffer as [col][row] halves, and leaves as VEC consecutive rows per lane:
// VEC = 8 (16-byte stores) for plain outputs, VEC = 4 (8-byte stores) when rows are re-spaced per window (t_row_group / t_row_pad
// multiples of 4 keep every 4-row run contiguous and 8-byte aligned).  Requires M % VEC == 0 and ldc % VEC == 0 (host-checked).
template <int VEC>
__device__ __forceinline__ void epilogue_transposed_f16(const GemmParams& p, const float* arow, uint32_t sbuf, int b, int m0, int n0,
                                                        int col_begin, int col_end, int lane) {
    __half* c_b = reinterpret_cast<__half*>(p.c_hi) + (int64_t)b * p.c_bstride;
    constexpr int SEGS = 32 / VEC;                  // row segments per column
    constexpr int ITER = 32 * SEGS / 32;            // (column, segment) items per lane
#pragma unroll 1
    for (int cb = col_begin; cb < col_end; cb += 32) {
        const int nbase = n0 + cb;
        if (nbase >= p.N) break;
        uint32_t v[32];
        acc_ld(arow + cb, v);
#pragma unroll
        for (int j = 0; j < 32; ++j) {
            float x = __uint_as_float(v[j]) * p.alpha;
            if (p.bias && nbase + j < p.N) x += __ldg(p.bias + nbase + j);
            const __half h = __float2half_rn(x);
            asm volatile("st.shared.u16 [%0], %1;" ::"r"(sbuf + (uint32_t)(j * 64 + lane * 2)), "h"(*reinterpret_cast<const unsigned short*>(&h)) : "memory");
        }
        __syncwarp();
#pragma unroll
        for (int i = 0; i < ITER; ++i) {
            const int idx = i * 32 + lane;
            const int cj = idx / SEGS, seg = idx - cj * SEGS;
            const int r = m0 + seg * VEC;
            const int col = nbase + cj;
            if (col < p.N && r < p.M) {
                const int row = p.t_row_group > 0 ? r + (r / p.t_row_group) * p.t_row_pad : r;
                __half* dst = c_b + (int64_t)col * p.ldc + row;
                if (VEC == 8) {
                    const float4 q = lds128(sbuf + (uint32_t)(cj * 64 + seg * 16));
                    *reinterpret_cast<float4*>(dst) = q;
                } else {
                    float2 q;
                    asm volatile("ld.shared.v2.f32 {%0,%1}, [%2];" : "=f"(q.x), "=f"(q.y) : "r"(sbuf + (uint32_t)(cj * 64 + seg * 8)) : "memory");
                    *reinterpret_cast<float2*>(dst) = q;
                }
            }
        }
        __syncwarp();
    }
}

// Transposed epilogue (C stored [col * ldc + row]): lanes hold 32 consecutive rows, so each register j is a
// coalesced 128-byte store along M; optional bit-packed (x > threshold) output packed along M.
__device__ __forceinline__ void epilogue_transposed(const GemmParams& p, const float* arow, int b, int m0, int n0,
                                                    int col_begin, int col_end, int lane) {
    const float* res_b = p.residual ? p.residual + (int64_t)b * p.r_bstride : nullptr;
    float* cf_b = p.c_f32 ? p.c_f32 + (int64_t)b * p.c_bstride : nullptr;
    __nv_bfloat16* chi_b = p.c_hi ? p.c_hi + (int64_t)b * p.c_bstride : nullptr;
    __nv_bfloat16* clo_b = p.c_lo ? p.c_lo + (int64_t)b * p.c_bstride : nullptr;
    const bool rok = m0 + lane < p.M;
    const int row = p.t_row_group > 0 ? (m0 + lane) + ((m0 + lane) / p.t_row_group) * p.t_row_pad : m0 + lane;
#pragma unroll 1
    for (int cb = col_begin; cb < col_end; cb += 32) {
        const int nbase = n0 + cb;
        if (nbase >= p.N) break;
        uint32_t v[32];
        acc_ld(arow + cb, v);
        uint32_t bitsword = 0;
#pragma unroll
        for (int j = 0; j < 32; ++j) {
            const int col = nbase + j;
            if (col < p.N) {
                float x = __uint_as_float(v[j]) * p.alpha;
                if (p.bias) x += __ldg(p.bias + col);
                x = act_apply(x, p.act);
                if (p.colscale) x *= __ldg(p.colscale + col);
                const int64_t off = (int64_t)col * p.ldc + row;
                if (res_b && rok) x += res_b[(int64_t)col * p.ldr + row];
                if (rok) {
                    if (cf_b) cf_b[off] = x;
                    if (chi_b) {
                        if (p.c_fp16) {
                            reinterpret_cast<__half*>(chi_b)[off] = __float2half_rn(x);
                        } else {
                            const __nv_bfloat16 h = __float2bfloat16_rn(x);
                            chi_b[off] = h;
                            if (clo_b) clo_b[off] = __float2bfloat16_rn(x - __bfloat162float(h));
                        }
                    }
                }
                if (p.c_bits) {
                    const uint32_t word = __ballot_sync(0xffffffffu, rok && x > p.bits_threshold);
                    if (lane == j) bitsword = word;
                }
            }
        }
        if (p.c_bits) {
            const int col = nbase + lane;
            if (col < p.N && m0 < p.M) {
                const int64_t words_per_col = (p.M + 31) / 32;
                p.c_bits[((int64_t)b * p.N + col) * words_per_col + (m0 >> 5)] = bitsword;
            }
        }
    }
}

// Row-major epilogue of the 128 x 256 tiles, straight from the wgmma register fragment (a staged fp32 copy of the tile would
// need 132 KB of shared memory).  The warp owns rows [m0, m0 + 16) and the 256 columns from n0.  Per 32-column chunk the two
// lanes of a pair swap half of their values (shfl.xor 1), so that every lane holds 4 consecutive columns of ONE row: lane
// 4 r + q holds row r + 8 (q & 1), columns 4 (q >> 1) + {0..3} of each 8-column group.  Bias, activation, layer-scale, residual
// and the output splits then run on float4s in the order of the staged epilogues above, so they write the same bits.
// Aligned outputs without a residual or row map leave as 16 x 32 TMA-store boxes, through the two 2 KB halves of the warp's
// staging buffer in turn (`half`); the others as 16-byte global stores, two lanes completing one 32-byte sector of a row.
// The chunk loop stays rolled (an unrolled one is ~8x the code, and the instruction fetch then bounds the GELU epilogue): each
// chunk reads acc[0, 16) and shifts the next chunk's values down, so every register index is a compile-time constant.
template <int ACT>
__device__ __forceinline__ void epilogue_frag(const GemmParams& p, const CUtensorMap* tm_f32, const CUtensorMap* tm_hi,
                                              const CUtensorMap* tm_lo, float (&acc)[128], uint32_t sbuf, uint32_t& half,
                                              int b, int m0, int n0, int lane) {
    if (m0 >= p.M) return;          // warp-uniform: these 16 rows lie below the matrix
    const int q = lane & 3, br = (lane >> 2) + 8 * (q & 1);     // row of this lane inside the 16-row box
    const bool odd = q & 1;
    const bool quick = p.act == HIPIE_ACT_QUICK_GELU;
    const float alpha = p.alpha;
    int64_t orow = -1;              // output row, -1: none (below the matrix, or a pad row of the row map)
    if (m0 + br < p.M) orow = p.row_map ? p.row_map[(int64_t)b * p.M + m0 + br] : m0 + br;
    const float* res_b = p.residual ? p.residual + (int64_t)b * p.r_bstride : nullptr;
    float* cf_b = p.c_f32 ? p.c_f32 + (int64_t)b * p.c_bstride : nullptr;
    __nv_bfloat16* chi_b = p.c_hi ? p.c_hi + (int64_t)b * p.c_bstride : nullptr;
    __nv_bfloat16* clo_b = p.c_lo ? p.c_lo + (int64_t)b * p.c_bstride : nullptr;
    const bool vec_ok = ((p.ldc & 3) == 0) && (!res_b || (p.ldr & 3) == 0);
#pragma unroll 1
    for (int ch = 0; ch < 8; ++ch) {
        const int nb = n0 + 32 * ch;
        if (nb >= p.N) break;       // warp-uniform
        float4 x[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int i = 4 * j;              // d[i + {0,1}]: row r, columns 2q + {0,1};  d[i + {2,3}]: row r + 8
            const float s0 = __shfl_xor_sync(0xffffffffu, odd ? acc[i] : acc[i + 2], 1);
            const float s1 = __shfl_xor_sync(0xffffffffu, odd ? acc[i + 1] : acc[i + 3], 1);
            x[j] = odd ? make_float4(s0, s1, acc[i + 2], acc[i + 3]) : make_float4(acc[i], acc[i + 1], s0, s1);
        }
#pragma unroll
        for (int i = 0; i < 112; ++i) acc[i] = acc[i + 16];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int col = nb + 8 * j + 4 * (q >> 1);
            const float4 bias = p.bias ? load4_guard(p.bias, col, p.N, 0.f) : make_float4(0.f, 0.f, 0.f, 0.f);
            x[j].x = act_apply_t<ACT>(fmaf(x[j].x, alpha, bias.x), quick);
            x[j].y = act_apply_t<ACT>(fmaf(x[j].y, alpha, bias.y), quick);
            x[j].z = act_apply_t<ACT>(fmaf(x[j].z, alpha, bias.z), quick);
            x[j].w = act_apply_t<ACT>(fmaf(x[j].w, alpha, bias.w), quick);
            if (p.colscale) {
                const float4 cs = load4_guard(p.colscale, col, p.N, 1.f);
                x[j].x *= cs.x; x[j].y *= cs.y; x[j].z *= cs.z; x[j].w *= cs.w;
            }
        }
        if (p.tma_out) {
            // f32 box: 128-byte rows, 16-byte group g of row r at g ^ (r & 7) (SWIZZLE_128B); fp16 / bf16 boxes: 64-byte rows, group c
            // of row r at c ^ ((r >> 1) & 3) (SWIZZLE_64B); the e4m3 box: 64-byte rows [slot 0 | slot 1] of the chunk, swizzled the same
#pragma unroll 1
            for (int pass = (p.c_f32 ? 0 : 1); pass < (p.c_hi ? 2 : 1); ++pass) {
                const uint32_t buf = sbuf + half * 2048;
                if (lane == 0) bulk_wait_read1();      // the store that last read this half has finished reading it
                __syncwarp();
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int g = 2 * j + (q >> 1);       // 4-column group inside the 32-column chunk
                    if (pass == 0) {
                        sts128(buf + br * 128 + ((g ^ (br & 7)) << 4), __float_as_uint(x[j].x), __float_as_uint(x[j].y),
                               __float_as_uint(x[j].z), __float_as_uint(x[j].w));
                        continue;
                    }
                    const uint32_t sw = (br >> 1) & 3, off = br * 64 + ((j ^ sw) << 4) + ((q >> 1) << 3);
                    uint2 hi, lo;
                    if (p.c_e4m3) {
                        uint32_t h8, l8;
                        split4_f16_e4m3(x[j], hi, h8, l8);
                        const uint32_t rb = buf + 1024 + br * 64 + 4 * (g & 3);
                        asm volatile("st.shared.b32 [%0], %1;" ::"r"(rb + ((((g >> 2)) ^ sw) << 4)), "r"(h8) : "memory");
                        asm volatile("st.shared.b32 [%0], %1;" ::"r"(rb + (((2 + (g >> 2)) ^ sw) << 4)), "r"(l8) : "memory");
                    } else {
                        split2m(x[j].x, x[j].y, hi.x, lo.x, p.c_fp16);
                        split2m(x[j].z, x[j].w, hi.y, lo.y, p.c_fp16);
                        if (p.c_lo) asm volatile("st.shared.v2.b32 [%0], {%1,%2};" ::"r"(buf + 1024 + off), "r"(lo.x), "r"(lo.y) : "memory");
                    }
                    asm volatile("st.shared.v2.b32 [%0], {%1,%2};" ::"r"(buf + off), "r"(hi.x), "r"(hi.y) : "memory");
                }
                fence_proxy_async_smem();      // generic-proxy writes -> visible to the TMA (async proxy)
                __syncwarp();
                if (lane == 0) {
                    if (pass == 0) {
                        tma_store_3d(tm_f32, buf, nb, m0, b);
                    } else {
                        tma_store_3d(tm_hi, buf, nb, m0, b);
                        if (p.c_e4m3) tma_store_3d(tm_lo, buf + 1024, 2 * nb, m0, b);      // both slots of columns [nb, nb + 32)
                        else if (p.c_lo) tma_store_3d(tm_lo, buf + 1024, nb, m0, b);
                    }
                    bulk_commit();
                }
                half ^= 1;
            }
            continue;
        }
        if (orow < 0) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int col = nb + 8 * j + 4 * (q >> 1);
            if (col >= p.N) continue;
            float4 v = x[j];
            const int64_t off = orow * p.ldc + col;
            if (col + 3 < p.N && vec_ok) {
                if (res_b) {
                    const float4 rv = *reinterpret_cast<const float4*>(res_b + orow * p.ldr + col);
                    v.x += rv.x; v.y += rv.y; v.z += rv.z; v.w += rv.w;
                }
                if (p.relu_post) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
                if (cf_b) *reinterpret_cast<float4*>(cf_b + off) = v;
                if (chi_b) {
                    uint2 hi, lo;
                    split2m(v.x, v.y, hi.x, lo.x, p.c_fp16);
                    split2m(v.z, v.w, hi.y, lo.y, p.c_fp16);
                    *reinterpret_cast<uint2*>(chi_b + off) = hi;
                    if (clo_b) *reinterpret_cast<uint2*>(clo_b + off) = lo;
                }
                continue;
            }
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                if (col + e >= p.N) break;
                float xv = e == 0 ? v.x : (e == 1 ? v.y : (e == 2 ? v.z : v.w));
                if (res_b) xv += res_b[orow * p.ldr + col + e];
                if (p.relu_post) xv = fmaxf(xv, 0.f);
                if (cf_b) cf_b[off + e] = xv;
                if (chi_b) {
                    if (p.c_fp16) {
                        reinterpret_cast<__half*>(chi_b)[off + e] = __float2half_rn(xv);
                    } else {
                        const __nv_bfloat16 h = __float2bfloat16_rn(xv);
                        chi_b[off + e] = h;
                        if (clo_b) clo_b[off + e] = __float2bfloat16_rn(xv - __bfloat162float(h));
                    }
                }
            }
        }
    }
}

// issue the wgmmas of one k-block for this warpgroup's 64 rows (A rows offset inside the stage by `a_off` bytes); F8: a k-block
// of the e4m3 sweep of prec 6
template <int PREC, int BN, bool F8>
__device__ __forceinline__ void gemm_kblock(float (&acc)[BN / 2], uint32_t st, uint32_t a_off, bool f16_ops, bool first) {
    using Cfg = GemmCfg<PREC, BN>;
    if constexpr (F8) {
        // e4m3 sweep: 128-byte rows, 32 bytes along K per wgmma
        const uint64_t da = wg::desc<128>(st + a_off), dw = wg::desc<128>(st + Cfg::A_TILE);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            if constexpr (BN == 256) wg::ss_e4m3_n256(acc, da + 2 * k, dw + 2 * k, !(first && k == 0));
            else if (BN == 64) wg::ss_e4m3_n64(*reinterpret_cast<float(*)[32]>(&acc), da + 2 * k, dw + 2 * k, !(first && k == 0));
            else wg::ss_e4m3_n128(*reinterpret_cast<float(*)[64]>(&acc), da + 2 * k, dw + 2 * k, !(first && k == 0));
        }
        return;
    }
    auto mma = [&](uint64_t da, uint64_t dw, int scale_d) {
        if constexpr (BN == 256) {
            wg::ss_f16_n256(acc, da, dw, scale_d);      // the wide tiles run prec 4 / 6: fp16 operands
        } else if (f16_ops) {
            if (BN == 64) wg::ss_f16_n64(*reinterpret_cast<float(*)[32]>(&acc), da, dw, scale_d);
            else wg::ss_f16_n128(*reinterpret_cast<float(*)[64]>(&acc), da, dw, scale_d);
        } else {
            if (BN == 64) wg::ss_bf16_n64(*reinterpret_cast<float(*)[32]>(&acc), da, dw, scale_d);
            else wg::ss_bf16_n128(*reinterpret_cast<float(*)[64]>(&acc), da, dw, scale_d);
        }
    };
    const uint64_t a_hi = wg::desc<Cfg::SWZ>(st + a_off), w_hi = wg::desc<Cfg::SWZ>(st + Cfg::A_TILE);
    // 16 elements (32 bytes) along K per wgmma inside the swizzle atom: +2 in addr>>4 units
#pragma unroll
    for (int k = 0; k < Cfg::BK / 16; ++k) mma(a_hi + 2 * k, w_hi + 2 * k, !(first && k == 0));
    if (Cfg::P4) {
        const uint64_t w_lo = wg::desc<Cfg::SWZ>(st + Cfg::A_TILE + Cfg::W_TILE);
#pragma unroll
        for (int k = 0; k < Cfg::BK / 16; ++k) mma(a_hi + 2 * k, w_lo + 2 * k, 1);
    }
    if (PREC == 3) {
        const uint64_t a_lo = wg::desc<Cfg::SWZ>(st + Cfg::A_TILE + Cfg::W_TILE + a_off);
        const uint64_t w_lo = wg::desc<Cfg::SWZ>(st + 2 * Cfg::A_TILE + Cfg::W_TILE);
#pragma unroll
        for (int k = 0; k < Cfg::BK / 16; ++k) mma(a_hi + 2 * k, w_lo + 2 * k, 1);
#pragma unroll
        for (int k = 0; k < Cfg::BK / 16; ++k) mma(a_lo + 2 * k, w_hi + 2 * k, 1);
    }
}

template <int PREC, int BN>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tm_a_hi, const __grid_constant__ CUtensorMap tm_a_lo,
               const __grid_constant__ CUtensorMap tm_w_hi, const __grid_constant__ CUtensorMap tm_w_lo,
               const __grid_constant__ CUtensorMap tm_c_f32, const __grid_constant__ CUtensorMap tm_c_hi,
               const __grid_constant__ CUtensorMap tm_c_lo, const GemmParams p) {
    using Cfg = GemmCfg<PREC, BN>;
    constexpr int BK = Cfg::BK;
    constexpr int STAGES = Cfg::STAGES;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // stays in the shared address space (LDS / STS)
    uint8_t* stage_base = smem;
    float* acc_s = reinterpret_cast<float*>(smem + STAGES * Cfg::STAGE);
    float* epi = reinterpret_cast<float*>(smem + STAGES * Cfg::STAGE + Cfg::ACC_BYTES);
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * Cfg::STAGE + Cfg::ACC_BYTES + Cfg::EPI_BYTES);
    uint64_t* full_bar = bars;                // [STAGES]
    uint64_t* empty_bar = bars + STAGES;      // [STAGES]  one arrival per consumer warp

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int num_kb8 = Cfg::P6 ? (2 * p.K + Cfg::BK8 - 1) / Cfg::BK8 : 0;     // k-blocks of the e4m3 sweep (planes are 2K wide)
    const int num_kb = num_kb8 + (p.K + BK - 1) / BK;
    const int tiles_per_batch = p.tiles_m * p.tiles_n;
    const int total_tiles = tiles_per_batch * p.batch;

    if (threadIdx.x == 0) {
        prefetch_tmap(&tm_a_hi);
        prefetch_tmap(&tm_w_hi);
        if (PREC == 3 || Cfg::P6) prefetch_tmap(&tm_a_lo);
        if (PREC == 3 || Cfg::P4 || Cfg::P6) prefetch_tmap(&tm_w_lo);
        for (int i = 0; i < STAGES; ++i) {
            mbar_init(&full_bar[i], 1);
            mbar_init(&empty_bar[i], GEMM_EPI_WARPS);
        }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp < 4) {
        // ===================== TMA producer (one thread) =====================
        if constexpr (Cfg::WIDE) setmaxnreg_dec<GEMM_PRODUCER_REGS>();
        if (threadIdx.x == 0) {
            int s = 0;
            uint32_t ph = 0;
            for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
                const int b = t / tiles_per_batch;
                const int r = t - b * tiles_per_batch;
                const int mt = p.m_fastest ? r % p.tiles_m : r / p.tiles_n, nt = p.m_fastest ? r / p.tiles_m : r - mt * p.tiles_n;
                const int m0 = mt * GEMM_BM, n0 = nt * BN;
                for (int kb = 0; kb < num_kb; ++kb) {
                    mbar_wait(&empty_bar[s], ph ^ 1);
                    uint8_t* st = stage_base + s * Cfg::STAGE;
                    mbar_arrive_expect_tx(&full_bar[s], Cfg::STAGE);
                    if (Cfg::P6 && kb < num_kb8) {
                        // sweep 1: e4m3 planes (maps tm_a_lo / tm_w_lo, 128-byte k-blocks); sweep 2: fp16 planes (64-element k-blocks)
                        tma_load_3d(st, &tm_a_lo, &full_bar[s], kb * Cfg::BK8, m0, b);
                        tma_load_3d(st + Cfg::A_TILE, &tm_w_lo, &full_bar[s], kb * Cfg::BK8, n0, b);
                    } else {
                        const int k0 = (kb - num_kb8) * BK;
                        tma_load_3d(st, &tm_a_hi, &full_bar[s], k0, m0, b);
                        tma_load_3d(st + Cfg::A_TILE, &tm_w_hi, &full_bar[s], k0, n0, b);
                        if (PREC == 3) {
                            tma_load_3d(st + Cfg::A_TILE + Cfg::W_TILE, &tm_a_lo, &full_bar[s], k0, m0, b);
                            tma_load_3d(st + 2 * Cfg::A_TILE + Cfg::W_TILE, &tm_w_lo, &full_bar[s], k0, n0, b);
                        }
                        if (Cfg::P4) tma_load_3d(st + Cfg::A_TILE + Cfg::W_TILE, &tm_w_lo, &full_bar[s], k0, n0, b);
                    }
                    if (++s == STAGES) { s = 0; ph ^= 1; }
                }
            }
        }
    } else {
        // ===================== consumer warpgroups: wgmma mainloop + epilogue =====================
        // warpgroup c owns rows [64 c, 64 c + 64) of the 128-row tile; the staged epilogue gives each of its warps 32 of those rows and
        // half of the BN columns, the wide one (epilogue_frag) the warp's 16 fragment rows and all 256 columns
        if constexpr (Cfg::WIDE) setmaxnreg_inc<GEMM_CONSUMER_REGS>();
        const int c = (threadIdx.x >> 7) - 1;
        const int wq = warp & 3;
        const int ew = warp - 4;                              // 0..7
        float* my_epi = epi + ew * (EPI_WARP_BYTES / 4);      // 4 KB per warp (1024-byte aligned: TMA swizzle atoms)
        const uint32_t my_sbuf = smem_u32(my_epi);
        float* acc_tile = acc_s + c * 64 * Cfg::ACC_LD;
        if (p.tma_out && lane == 0) {
            if (p.c_f32) prefetch_tmap(&tm_c_f32);
            if (p.c_hi) prefetch_tmap(&tm_c_hi);
            if (p.c_lo || p.c_e4m3) prefetch_tmap(&tm_c_lo);
        }
        constexpr int COLS_PER = BN / 2;                      // columns per epilogue warp (a multiple of the 32-column chunk)
        const int cbeg = (wq >> 1) * COLS_PER, cend = cbeg + COLS_PER;
        const uint32_t a_off = (uint32_t)c * 64u * (uint32_t)Cfg::SWZ;            // 64 rows of the 16-bit A tile
        const uint32_t a_off8 = (uint32_t)c * 64u * (uint32_t)Cfg::BK8;           // ... of the e4m3 A tile
        int s = 0;
        uint32_t ph = 0;
        uint32_t half = 0;                                    // epilogue_frag: staging half of the next TMA-store box
        for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
            const int b = t / tiles_per_batch;
            const int r = t - b * tiles_per_batch;
            const int mt = p.m_fastest ? r % p.tiles_m : r / p.tiles_n, nt = p.m_fastest ? r / p.tiles_m : r - mt * p.tiles_n;
            float acc[BN / 2];
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
            int prev = -1;
            auto kblock = [&](auto f8, bool first) {
                mbar_wait(&full_bar[s], ph);
                wg::fence_regs(acc);
                wg::fence();
                gemm_kblock<PREC, BN, decltype(f8)::value>(acc, smem_u32(stage_base + s * Cfg::STAGE), f8 ? a_off8 : a_off, p.f16_ops != 0, first);
                wg::commit();
                wg::wait<1>();                                   // the previous k-block's wgmmas have read their stage
                wg::fence_regs(acc);
                if (prev >= 0) {
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&empty_bar[prev]);
                }
                prev = s;
                if (++s == STAGES) { s = 0; ph ^= 1; }
            };
            // two loops, so that no wgmma and no accumulator update sits under a condition: ptxas serialises every wgmma of the
            // kernel otherwise
            if constexpr (Cfg::P6) {
                for (int kb = 0; kb < num_kb8; ++kb) kblock(std::true_type{}, kb == 0);
                // the e4m3 sweep accumulated 2^14 x the cross terms: rescale before the fp16 sweep adds Ah.Wh
                wg::wait<0>();
                wg::fence_regs(acc);
#pragma unroll
                for (int i = 0; i < BN / 2; ++i) acc[i] *= 0x1p-14f;
            }
            for (int kb = num_kb8; kb < num_kb; ++kb) kblock(std::false_type{}, kb == 0);
            wg::wait<0>();
            wg::fence_regs(acc);
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[prev]);
            if constexpr (Cfg::WIDE) {
                const int m0 = mt * GEMM_BM + c * 64 + wq * 16, n0 = nt * BN;
                switch (p.act) {
                    case HIPIE_ACT_RELU: epilogue_frag<HIPIE_ACT_RELU>(p, &tm_c_f32, &tm_c_hi, &tm_c_lo, acc, my_sbuf, half, b, m0, n0, lane); break;
                    case HIPIE_ACT_GELU: epilogue_frag<HIPIE_ACT_GELU>(p, &tm_c_f32, &tm_c_hi, &tm_c_lo, acc, my_sbuf, half, b, m0, n0, lane); break;
                    case HIPIE_ACT_QUICK_GELU:
                    case HIPIE_ACT_SIGMOID: epilogue_frag<HIPIE_ACT_SIGMOID>(p, &tm_c_f32, &tm_c_hi, &tm_c_lo, acc, my_sbuf, half, b, m0, n0, lane); break;
                    default: epilogue_frag<HIPIE_ACT_NONE>(p, &tm_c_f32, &tm_c_hi, &tm_c_lo, acc, my_sbuf, half, b, m0, n0, lane); break;
                }
                continue;
            }
            // accumulator fragment -> staged tile (row-major, padded): d[4j + {0,1}] at (16 wq + lane / 4, 8 j + 2 (lane % 4)), +8 rows
            {
                const int r0 = 16 * wq + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
                for (int j = 0; j < BN / 8; ++j) {
                    *reinterpret_cast<float2*>(acc_tile + r0 * Cfg::ACC_LD + 8 * j + c0) = make_float2(acc[4 * j], acc[4 * j + 1]);
                    *reinterpret_cast<float2*>(acc_tile + (r0 + 8) * Cfg::ACC_LD + 8 * j + c0) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
                }
            }
            named_bar_sync(1 + c, 128);
            const int m0 = mt * GEMM_BM + c * 64 + (wq & 1) * 32, n0 = nt * BN;
            const float* arow = acc_tile + ((wq & 1) * 32 + lane) * Cfg::ACC_LD;
            if (m0 - (wq & 1) * 32 < p.M) {
                if (p.transposed == 2)
                    epilogue_transposed_f16<8>(p, arow, my_sbuf, b, m0, n0, cbeg, cend, lane);
                else if (p.transposed == 3)
                    epilogue_transposed_f16<4>(p, arow, my_sbuf, b, m0, n0, cbeg, cend, lane);
                else if (p.transposed)
                    epilogue_transposed(p, arow, b, m0, n0, cbeg, cend, lane);
                else if (p.tma_out)
                    switch (p.act) {
                        case HIPIE_ACT_RELU: epilogue_rows_tma<HIPIE_ACT_RELU>(p, &tm_c_f32, &tm_c_hi, &tm_c_lo, arow, my_sbuf, b, m0, n0, cbeg, cend, lane); break;
                        case HIPIE_ACT_GELU: epilogue_rows_tma<HIPIE_ACT_GELU>(p, &tm_c_f32, &tm_c_hi, &tm_c_lo, arow, my_sbuf, b, m0, n0, cbeg, cend, lane); break;
                        case HIPIE_ACT_QUICK_GELU:
                        case HIPIE_ACT_SIGMOID: epilogue_rows_tma<HIPIE_ACT_SIGMOID>(p, &tm_c_f32, &tm_c_hi, &tm_c_lo, arow, my_sbuf, b, m0, n0, cbeg, cend, lane); break;
                        default: epilogue_rows_tma<HIPIE_ACT_NONE>(p, &tm_c_f32, &tm_c_hi, &tm_c_lo, arow, my_sbuf, b, m0, n0, cbeg, cend, lane); break;
                    }
                else
                    switch (p.act) {
                        case HIPIE_ACT_RELU: epilogue_rows<HIPIE_ACT_RELU>(p, arow, my_epi, b, m0, n0, cbeg, cend, lane); break;
                        case HIPIE_ACT_GELU: epilogue_rows<HIPIE_ACT_GELU>(p, arow, my_epi, b, m0, n0, cbeg, cend, lane); break;
                        case HIPIE_ACT_QUICK_GELU:
                        case HIPIE_ACT_SIGMOID: epilogue_rows<HIPIE_ACT_SIGMOID>(p, arow, my_epi, b, m0, n0, cbeg, cend, lane); break;
                        default: epilogue_rows<HIPIE_ACT_NONE>(p, arow, my_epi, b, m0, n0, cbeg, cend, lane); break;
                    }
            }
            named_bar_sync(1 + c, 128);                       // the staged tile is read out before the next tile overwrites it
        }
        if (p.tma_out && lane == 0) bulk_wait0();     // outstanding TMA stores read this CTA's shared memory
    }
}

// ------------------------------------------------------------------------------------------
// host side: tensor-map construction (driver entry point fetched through the runtime) + launch
// ------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* f = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(f);
    });
    return fn;
}

struct TmapKey {
    const void* ptr;
    int64_t rows, cols, ld, bstride;
    int batch, box_rows, box_cols, esize, pad_;
    bool operator==(const TmapKey& o) const { return memcmp(this, &o, sizeof(TmapKey)) == 0; }
};
struct TmapKeyHash {
    size_t operator()(const TmapKey& k) const {
        const uint64_t* w = reinterpret_cast<const uint64_t*>(&k);
        uint64_t h = 1469598103934665603ull;
        for (size_t i = 0; i < sizeof(TmapKey) / 8; ++i) { h ^= w[i]; h *= 1099511628211ull; }
        return (size_t)h;
    }
};

// bf16 matrix (batch, rows, cols) with row stride ld and batch stride bstride (elements);
// box = (box_cols along K, box_rows, 1); swizzle span == box_cols*2 bytes.
int make_tmap(CUtensorMap* out, const void* ptr, int esize, int64_t rows, int64_t cols, int64_t ld, int batch, int64_t bstride,
              int box_rows, int box_cols);

int make_tmap_bf16(CUtensorMap* out, const void* ptr, int64_t rows, int64_t cols, int64_t ld, int batch,
                   int64_t bstride, int box_rows, int box_cols) {
    return make_tmap(out, ptr, 2, rows, cols, ld, batch, bstride, box_rows, box_cols);
}

// matrix (batch, rows, cols) of 1-byte (e4m3), 2-byte (bf16 / fp16) or 4-byte (fp32) elements; swizzle span == box_cols * esize bytes (32 / 64 / 128)
int make_tmap(CUtensorMap* out, const void* ptr, int esize, int64_t rows, int64_t cols, int64_t ld, int batch, int64_t bstride,
              int box_rows, int box_cols) {
    static std::mutex mu;
    static std::unordered_map<TmapKey, CUtensorMap, TmapKeyHash> cache;
    TmapKey key;
    memset(&key, 0, sizeof(key));
    key.ptr = ptr; key.rows = rows; key.cols = cols; key.ld = ld; key.bstride = bstride;
    key.batch = batch; key.box_rows = box_rows; key.box_cols = box_cols; key.esize = esize;
    {
        std::lock_guard<std::mutex> g(mu);
        auto it = cache.find(key);
        if (it != cache.end()) { *out = it->second; return HIPIE_OK; }
    }
    EncodeTiledFn enc = get_encode_fn();
    if (!enc) { set_error("cuTensorMapEncodeTiled entry point unavailable"); return HIPIE_ECUDA; }
    HIPIE_CHECK_ARG((reinterpret_cast<uintptr_t>(ptr) & 15) == 0, "tensor map base %p not 16B aligned", ptr);
    HIPIE_CHECK_ARG((ld * esize) % 16 == 0, "row stride %lld elements is not a multiple of 16 bytes", (long long)ld);
    HIPIE_CHECK_ARG(batch == 1 || (bstride * esize) % 16 == 0, "batch stride must be a multiple of 16 bytes");
    cuuint64_t dims[3] = {(cuuint64_t)cols, (cuuint64_t)rows, (cuuint64_t)batch};
    cuuint64_t strides[2] = {(cuuint64_t)ld * esize, (cuuint64_t)(batch > 1 ? bstride : rows * ld) * esize};
    cuuint32_t box[3] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    CUtensorMapSwizzle swz = box_cols * esize == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                             : (box_cols * esize == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
    const CUtensorMapDataType dt = esize == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : (esize == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16);
    CUresult r = enc(out, dt, 3, const_cast<void*>(ptr), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled failed (%d): ptr=%p rows=%lld cols=%lld ld=%lld batch=%d", (int)r, ptr,
                  (long long)rows, (long long)cols, (long long)ld, batch);
        return HIPIE_ECUDA;
    }
    {
        std::lock_guard<std::mutex> g(mu);
        if (cache.size() > 4096) cache.clear();
        cache.emplace(key, *out);
    }
    return HIPIE_OK;
}

// hipie_set_option switches (A/B measurements, fallbacks): TMA-store epilogue
int g_gemm_tma_store = 1;
int g_gemm_fast_transposed = 1;   // vectorised fp16-plane transposed epilogue (A/B switch)

// fp32 tensor of rank 5 (dims / strides innermost first, strides in BYTES for dims 1..4), dense unswizzled boxes: the value-map
// windows of the shared-memory MSDeformAttn kernel (msda.cu).  Not cached: built once per launch from host-side geometry.
int make_tmap_f32_5d(CUtensorMap* out, const void* ptr, const uint64_t dims[5], const uint64_t strides_bytes[4], const uint32_t box[5]) {
    EncodeTiledFn enc = get_encode_fn();
    if (!enc) { set_error("cuTensorMapEncodeTiled entry point unavailable"); return HIPIE_ECUDA; }
    HIPIE_CHECK_ARG((reinterpret_cast<uintptr_t>(ptr) & 15) == 0, "tensor map base %p not 16B aligned", ptr);
    cuuint64_t d[5], st[4];
    cuuint32_t bx[5], es[5] = {1, 1, 1, 1, 1};
    for (int i = 0; i < 5; ++i) { d[i] = dims[i]; bx[i] = box[i]; }
    for (int i = 0; i < 4; ++i) {
        HIPIE_CHECK_ARG(strides_bytes[i] % 16 == 0, "tensor map stride %llu not a multiple of 16 bytes", (unsigned long long)strides_bytes[i]);
        st[i] = strides_bytes[i];
    }
    CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 5, const_cast<void*>(ptr), d, st, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled (5-d) failed (%d): dims %llu %llu %llu %llu %llu box %u %u %u %u %u", (int)r, (unsigned long long)d[0],
                  (unsigned long long)d[1], (unsigned long long)d[2], (unsigned long long)d[3], (unsigned long long)d[4], bx[0], bx[1], bx[2],
                  bx[3], bx[4]);
        return HIPIE_ECUDA;
    }
    return HIPIE_OK;
}

template <int PREC, int BN>
static int launch_gemm(const hipie_gemm_args* a, cudaStream_t st) {
    using Cfg = GemmCfg<PREC, BN>;
    CUtensorMap ta_hi, ta_lo, tw_hi, tw_lo;
    int rc;
    if ((rc = make_tmap_bf16(&ta_hi, a->a_hi, a->M, a->K, a->lda, a->batch, a->a_bstride, GEMM_BM, Cfg::BK))) return rc;
    if ((rc = make_tmap_bf16(&tw_hi, a->w_hi, a->N, a->K, a->ldw, a->batch, a->w_bstride, BN, Cfg::BK))) return rc;
    ta_lo = ta_hi;
    tw_lo = tw_hi;
    if (Cfg::P6) {       // e4m3 planes, 2K wide, 128-byte k-blocks
        if ((rc = make_tmap(&ta_lo, a->a8, 1, a->M, 2 * (int64_t)a->K, a->lda8, 1, 0, GEMM_BM, Cfg::BK8))) return rc;
        if ((rc = make_tmap(&tw_lo, a->w8, 1, a->N, 2 * (int64_t)a->K, a->ldw8, 1, 0, BN, Cfg::BK8))) return rc;
    }
    if (PREC == 3 && (rc = make_tmap_bf16(&ta_lo, a->a_lo, a->M, a->K, a->lda, a->batch, a->a_bstride, GEMM_BM, Cfg::BK))) return rc;
    if ((PREC == 3 || Cfg::P4) &&
        (rc = make_tmap_bf16(&tw_lo, a->w_lo, a->N, a->K, a->ldw, a->batch, a->w_bstride, BN, Cfg::BK))) return rc;
    // row-major outputs through TMA stores when nothing needs per-element addressing (residual / row map / transposed stay on the
    // register path) and the output rows satisfy TMA's 16-byte rules
    auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
    bool tma_out = g_gemm_tma_store && !a->transposed && !a->c_row_map && !a->residual && al16(a->bias) && al16(a->colscale);
    if (a->c_f32) tma_out = tma_out && al16(a->c_f32) && (a->ldc * 4) % 16 == 0 && (a->batch == 1 || (a->c_bstride * 4) % 16 == 0);
    if (a->c_hi) tma_out = tma_out && al16(a->c_hi) && (!a->c_lo || al16(a->c_lo)) && (a->ldc * 2) % 16 == 0 &&
                           (a->batch == 1 || (a->c_bstride * 2) % 16 == 0);
    if (!a->c_f32 && !a->c_hi) tma_out = false;
    HIPIE_CHECK_ARG(!a->c8 || tma_out, "hipie_gemm: the e4m3 output planes (c8) need the TMA-store epilogue (row-major, no residual / row map, aligned)");
    CUtensorMap tc_f32 = ta_hi, tc_hi = ta_hi, tc_lo = ta_hi;
    if (tma_out) {
        const int64_t cbs = a->batch > 1 ? a->c_bstride : (int64_t)a->M * a->ldc;
        const int box_rows = Cfg::WIDE ? 16 : 32;      // rows per epilogue warp
        if (a->c_f32 && (rc = make_tmap(&tc_f32, a->c_f32, 4, a->M, a->N, a->ldc, a->batch, cbs, box_rows, 32))) return rc;
        if (a->c_hi && (rc = make_tmap(&tc_hi, a->c_hi, 2, a->M, a->N, a->ldc, a->batch, cbs, box_rows, 32))) return rc;
        if (a->c_lo && (rc = make_tmap(&tc_lo, a->c_lo, 2, a->M, a->N, a->ldc, a->batch, cbs, box_rows, 32))) return rc;
        if (a->c8 && (rc = make_tmap(&tc_lo, a->c8, 1, a->M, 2 * (int64_t)a->N, a->ldc8, 1, 0, box_rows, 64))) return rc;
    }
    GemmParams p;
    p.tma_out = tma_out ? 1 : 0;
    p.c_fp16 = a->c_fp16 ? 1 : 0;
    p.c_e4m3 = a->c8 ? 1 : 0;
    p.relu_post = a->relu_after_residual ? 1 : 0;
    p.f16_ops = (a->prec == 2 || a->prec == 4 || a->prec == 6) ? 1 : 0;
    p.bias = a->bias; p.colscale = a->colscale; p.residual = a->residual;
    p.ldr = a->ldr; p.r_bstride = a->r_bstride;
    p.c_f32 = a->c_f32; p.c_hi = (__nv_bfloat16*)a->c_hi; p.c_lo = (__nv_bfloat16*)a->c_lo;
    p.ldc = a->ldc; p.c_bstride = a->c_bstride;
    p.c_bits = a->c_bits; p.bits_threshold = a->bits_threshold;
    p.M = a->M; p.N = a->N; p.K = a->K; p.batch = a->batch;
    p.act = a->act; p.alpha = a->alpha;
    p.transposed = a->transposed;
    if (a->transposed && a->c_fp16 && a->c_hi && !a->c_f32 && !a->c_lo && !a->c_bits && !a->residual && !a->colscale && a->act == HIPIE_ACT_NONE &&
        g_gemm_fast_transposed && (reinterpret_cast<uintptr_t>(a->c_hi) & 15) == 0) {
        // vectorised V^T epilogue: whole 8-row (or, with per-window row padding, 4-row) runs must exist and stay aligned
        const bool grp4 = a->t_row_group > 0 && a->t_row_group % 4 == 0 && a->t_row_pad % 4 == 0;
        if (a->t_row_group == 0 && a->M % 8 == 0 && a->ldc % 8 == 0 && (a->batch == 1 || a->c_bstride % 8 == 0)) p.transposed = 2;
        else if ((grp4 || a->t_row_group == 0) && a->M % 4 == 0 && a->ldc % 4 == 0 && (a->batch == 1 || a->c_bstride % 4 == 0)) p.transposed = 3;
    }
    p.row_map = a->c_row_map;
    p.t_row_group = a->transposed ? a->t_row_group : 0;
    p.t_row_pad = a->transposed ? a->t_row_pad : 0;
    p.tiles_m = (a->M + GEMM_BM - 1) / GEMM_BM;
    p.tiles_n = (a->N + BN - 1) / BN;
    p.m_fastest = (p.tiles_m <= 8 && p.tiles_n >= 4 * p.tiles_m) ? 1 : 0;
    const int64_t total = (int64_t)p.tiles_m * p.tiles_n * a->batch;
    HIPIE_ENSURE_SMEM((gemm_tc_kernel<PREC, BN>), Cfg::SMEM);
    const int units = num_sms();      // persistent: one CTA per SM
    const int grid = (int)(total < units ? total : units);
    gemm_tc_kernel<PREC, BN><<<grid, GEMM_THREADS, Cfg::SMEM, st>>>(ta_hi, ta_lo, tw_hi, tw_lo, tc_f32, tc_hi, tc_lo, p);
    HIPIE_CHECK_LAUNCH();
    return HIPIE_OK;
}

}  // namespace hipie

using namespace hipie;

extern "C" int hipie_gemm(const hipie_gemm_args* a, void* stream) {
    HIPIE_CHECK_ARG(a != nullptr, "hipie_gemm: null args");
    HIPIE_CHECK_ARG(a->a_hi && a->w_hi, "hipie_gemm: a_hi / w_hi required");
    HIPIE_CHECK_ARG((a->prec >= 1 && a->prec <= 4) || a->prec == 6, "hipie_gemm: prec must be 1, 2, 3, 4 or 6 (got %d)", a->prec);
    HIPIE_CHECK_ARG(a->prec != 6 || a->K % 32 == 0, "hipie_gemm: prec 6 needs K %% 32 == 0 (the e4m3 planes interleave 32-column groups)");
    HIPIE_CHECK_ARG(a->prec != 6 || (!a->transposed && !a->c_bits), "hipie_gemm: prec 6 writes row-major outputs without the bit-packed mask");
    HIPIE_CHECK_ARG(a->prec != 6 || (a->a8 && a->w8 && a->batch == 1 && a->lda8 % 16 == 0 && a->ldw8 % 16 == 0 && a->lda8 >= 2 * (int64_t)a->K &&
                                     a->ldw8 >= 2 * (int64_t)a->K),
                    "hipie_gemm: prec 6 needs the e4m3 planes a8 (M x 2K) / w8 (N x 2K) with 16-byte aligned row strides, batch 1");
    HIPIE_CHECK_ARG(!a->c8 || (a->c_fp16 && a->c_hi && !a->c_lo && a->N % 32 == 0 && a->batch == 1 && a->ldc8 % 16 == 0 && a->ldc8 >= 2 * (int64_t)a->N),
                    "hipie_gemm: c8 (e4m3 planes of the result) goes with c_fp16, N %% 32 == 0, batch 1 and a 16-byte aligned ldc8 >= 2N");
    HIPIE_CHECK_ARG(a->prec != 3 || (a->a_lo && a->w_lo), "hipie_gemm: prec 3 needs a_lo and w_lo");
    HIPIE_CHECK_ARG(a->prec != 4 || a->w_lo, "hipie_gemm: prec 4 (A fp16, W fp16 hi + lo) needs w_lo");
    HIPIE_CHECK_ARG(a->M > 0 && a->N > 0 && a->K > 0 && a->batch > 0, "hipie_gemm: bad sizes M=%d N=%d K=%d batch=%d",
                    a->M, a->N, a->K, a->batch);
    HIPIE_CHECK_ARG(a->K % 8 == 0, "hipie_gemm: K (%d) must be a multiple of 8", a->K);
    HIPIE_CHECK_ARG(a->c_f32 || a->c_hi || a->c_bits, "hipie_gemm: no output requested");
    HIPIE_CHECK_ARG(!a->c_bits || a->transposed || (a->N % 16 == 0 && !a->c_row_map),
                    "hipie_gemm: row-major bit-packed output needs N %% 16 == 0 and no row map");
    HIPIE_CHECK_ARG(!a->c_lo || a->c_hi, "hipie_gemm: c_lo requires c_hi");
    HIPIE_CHECK_ARG(!a->relu_after_residual || (a->residual && !a->transposed), "hipie_gemm: relu_after_residual needs a row-major residual");
    HIPIE_CHECK_ARG(!a->c_fp16 || (a->c_hi && !a->c_lo), "hipie_gemm: c_fp16 writes one fp16 plane (c_hi set, c_lo NULL)");
    HIPIE_CHECK_ARG(!a->c_row_map || !a->transposed, "hipie_gemm: c_row_map is not supported with transposed=1");
    cudaStream_t st = (cudaStream_t)stream;
    // 128 x 64 tiles for narrow outputs, 128 x 128 otherwise (the fp32 accumulator of a 64-row warpgroup is 64 registers per
    // thread at N = 128; its staged copy for the epilogue is what bounds the tile width in shared memory).  The ViT linears run
    // 128 x 256 tiles with the epilogue from registers: a quarter fewer operand bytes per flop, which is what feeds the tensor
    // cores from L2 at these shapes.  prec 6 (row-major only) takes them for every N > 64, ragged N clipped by the TMA; prec 4
    // keeps 128 x 128 for N < 256, the transposed V^T output and the bit-packed mask.
    const bool narrow = a->N <= 64;
    if (a->prec == 6) return narrow ? launch_gemm<6, 64>(a, st) : launch_gemm<6, 256>(a, st);   // fp16 + e4m3 split (the large ViT linears)
    if (a->prec == 4) {                                                                           // two-pass fp16 (the qkv linears)
        if (narrow) return launch_gemm<4, 64>(a, st);
        return (a->N >= 256 && !a->transposed && !a->c_bits) ? launch_gemm<4, 256>(a, st) : launch_gemm<4, 128>(a, st);
    }
    // prec 1 (bf16) and prec 2 (fp16) share the single-plane kernels; the wgmma type differs
    if (a->prec == 3) return narrow ? launch_gemm<3, 64>(a, st) : launch_gemm<3, 128>(a, st);
    return narrow ? launch_gemm<1, 64>(a, st) : launch_gemm<1, 128>(a, st);
}

extern int g_ln_grid_cap, g_ln_bulk;          // norm.cu (global scope)
extern "C" int hipie_set_option(const char* name, int value) {
    HIPIE_CHECK_ARG(name != nullptr, "hipie_set_option: null name");
    if (strcmp(name, "gemm_tma_store") == 0) { g_gemm_tma_store = value ? 1 : 0; return HIPIE_OK; }
    if (strcmp(name, "gemm_fast_transposed") == 0) { g_gemm_fast_transposed = value ? 1 : 0; return HIPIE_OK; }
    if (strcmp(name, "ln_grid_cap") == 0) { g_ln_grid_cap = value ? 1 : 0; return HIPIE_OK; }
    if (strcmp(name, "ln_bulk") == 0) { g_ln_bulk = value ? 1 : 0; return HIPIE_OK; }
    set_error("hipie_set_option: unknown option '%s'", name);
    return HIPIE_EINVAL;
}
