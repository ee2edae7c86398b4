// Fused multi-head attention (flash-style online softmax; the (T x T) score matrix never exists
// in HBM) with the ViTDet decomposed relative-position bias and an optional additive key bias.
//
// Reference semantics: softmax((q*scale) k^T + rel_h[q, kh] + rel_w[q, kw]) v
//   (/root/reference/projects/HIPIE/hipie/backbone/vit.py:67-83, backbone/utils.py:96-125),
// nn.MultiheadAttention of the decoders (deformable_transformer_dino.py:432-438) and BERT
// self-attention with a padding mask (key_bias).
//
// Round-1 implementation: warp-level mma.sync (m16n8k16 bf16, fp32 accumulate) with cp.async
// double-buffered K/V tiles.  Operands are bf16 hi/lo planes; prec==3 evaluates
// S = Qh.Kh + Qh.Kl + Ql.Kh and O += Ph.Vh + Ph.Vl + Pl.Vh so the result is fp32-class.
#include "common.cuh"

namespace hipie {

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
                 : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
                 : "r"(addr));
}
__device__ __forceinline__ void mma_bf16(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void mma_f16(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
template <bool F16>
__device__ __forceinline__ void mma_16b(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    if (F16) mma_f16(c, a, b0, b1);
    else mma_bf16(c, a, b0, b1);
}
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, int src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

struct AttnParams {
    const __nv_bfloat16 *q_hi, *q_lo, *k_hi, *k_lo, *v_hi, *v_lo;
    int64_t q_bs, q_ts, q_hs, k_bs, k_ts, k_hs, v_bs, v_ts, v_hs;
    const float *rel_h, *rel_w;
    int kh, kw;
    const float* key_bias;
    const uint32_t* key_mask;     // (B, Tq, ceil(Tk/32)) bit words: bit set = key masked out for that query, or null
    float* out_f32;
    __nv_bfloat16 *out_hi, *out_lo;
    int64_t o_bs, o_ts;
    int B, H, Tq, Tk;
    float scale;
};

constexpr int ATT_BM = 64;   // query rows per CTA (4 warps x 16)
constexpr int ATT_BN = 64;   // keys per tile

template <int HD, int PREC>
__global__ void __launch_bounds__(128)
attention_kernel(const AttnParams p) {
    constexpr int ROWB = HD * 2 + 16;             // padded smem row (bytes), odd number of 16B units
    constexpr int PLANE = ATT_BN * ROWB;          // one K or V plane of a tile
    constexpr int NPL = PREC == 3 ? 4 : 2;        // Khi,(Klo),Vhi,(Vlo)
    constexpr int STAGE = NPL * PLANE;
    constexpr int KSTEPS = HD / 16;
    constexpr int DTILES = HD / 8;
    constexpr int CHUNKS = HD / 8;                // 16B chunks per row
    extern __shared__ __align__(16) uint8_t smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int q0 = blockIdx.x * ATT_BM;
    const int h = blockIdx.y, b = blockIdx.z;
    const uint32_t smem_base = (uint32_t)__cvta_generic_to_shared(smem);

    const __nv_bfloat16* qh_g = p.q_hi + (int64_t)b * p.q_bs + (int64_t)h * p.q_hs;
    const __nv_bfloat16* ql_g = PREC == 3 ? p.q_lo + (int64_t)b * p.q_bs + (int64_t)h * p.q_hs : nullptr;
    const __nv_bfloat16* kv_g[4];
    int64_t kv_ts[4];
    kv_g[0] = p.k_hi + (int64_t)b * p.k_bs + (int64_t)h * p.k_hs; kv_ts[0] = p.k_ts;
    if (PREC == 3) {
        kv_g[1] = p.k_lo + (int64_t)b * p.k_bs + (int64_t)h * p.k_hs; kv_ts[1] = p.k_ts;
        kv_g[2] = p.v_hi + (int64_t)b * p.v_bs + (int64_t)h * p.v_hs; kv_ts[2] = p.v_ts;
        kv_g[3] = p.v_lo + (int64_t)b * p.v_bs + (int64_t)h * p.v_hs; kv_ts[3] = p.v_ts;
    } else {
        kv_g[1] = p.v_hi + (int64_t)b * p.v_bs + (int64_t)h * p.v_hs; kv_ts[1] = p.v_ts;
        kv_g[2] = kv_g[3] = nullptr; kv_ts[2] = kv_ts[3] = 0;
    }
    constexpr int VPL = PREC == 3 ? 2 : 1;  // index of the first V plane

    auto load_tile = [&](int stage, int kv0) {
        const uint32_t sb = smem_base + stage * STAGE;
#pragma unroll
        for (int pl = 0; pl < NPL; ++pl) {
            for (int i = threadIdx.x; i < ATT_BN * CHUNKS; i += 128) {
                const int r = i / CHUNKS, c = i - r * CHUNKS;
                const int key = kv0 + r;
                const bool ok = key < p.Tk;
                const __nv_bfloat16* src = kv_g[pl] + (int64_t)(ok ? key : 0) * kv_ts[pl] + c * 8;
                cp_async16(sb + pl * PLANE + r * ROWB + c * 16, src, ok ? 16 : 0);
            }
        }
    };

    // ---- stage Q (hi, lo) through the second stage buffer, pull A fragments into registers ----
    {
        const uint32_t sb = smem_base + STAGE;
        for (int pl = 0; pl < (PREC == 3 ? 2 : 1); ++pl) {
            const __nv_bfloat16* g = pl == 0 ? qh_g : ql_g;
            for (int i = threadIdx.x; i < ATT_BM * CHUNKS; i += 128) {
                const int r = i / CHUNKS, c = i - r * CHUNKS;
                const int q = q0 + r;
                const bool ok = q < p.Tq;
                cp_async16(sb + pl * PLANE + r * ROWB + c * 16, g + (int64_t)(ok ? q : 0) * p.q_ts + c * 8, ok ? 16 : 0);
            }
        }
        cp_async_commit();
    }
    load_tile(0, 0);
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    uint32_t qa_hi[KSTEPS][4], qa_lo[PREC == 3 ? KSTEPS : 1][4];
    {
        const uint32_t sb = smem_base + STAGE;
        const int r = warp * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
        const int cb = (lane >> 4) * 16;  // bytes
#pragma unroll
        for (int kk = 0; kk < KSTEPS; ++kk) {
            ldsm_x4(sb + r * ROWB + kk * 32 + cb, qa_hi[kk][0], qa_hi[kk][1], qa_hi[kk][2], qa_hi[kk][3]);
            if (PREC == 3)
                ldsm_x4(sb + PLANE + r * ROWB + kk * 32 + cb, qa_lo[kk][0], qa_lo[kk][1], qa_lo[kk][2], qa_lo[kk][3]);
        }
    }
    __syncthreads();

    float o[DTILES][4];
#pragma unroll
    for (int j = 0; j < DTILES; ++j) o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    const int qrow[2] = {q0 + warp * 16 + (lane >> 2), q0 + warp * 16 + (lane >> 2) + 8};
    const bool has_rel = p.rel_h != nullptr;
    const float* relh_r[2] = {nullptr, nullptr};
    const float* relw_r[2] = {nullptr, nullptr};
    if (has_rel) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int qq = min(qrow[i], p.Tq - 1);
            relh_r[i] = p.rel_h + (((int64_t)b * p.H + h) * p.Tq + qq) * p.kh;
            relw_r[i] = p.rel_w + (((int64_t)b * p.H + h) * p.Tq + qq) * p.kw;
        }
    }
    const float* kb = p.key_bias ? p.key_bias + (int64_t)b * p.Tk : nullptr;
    const int mask_words = (p.Tk + 31) / 32;
    const uint32_t* km_r[2] = {nullptr, nullptr};      // this thread's two query rows of the boolean attention mask
    if (p.key_mask) {
#pragma unroll
        for (int i = 0; i < 2; ++i) km_r[i] = p.key_mask + ((int64_t)b * p.Tq + min(qrow[i], p.Tq - 1)) * mask_words;
    }
    // one KV tile == one key row of the grid (kw == 64): rel_w terms are tile-invariant -> registers
    const bool hoist = has_rel && p.kw == ATT_BN;
    // otherwise (14x14 windows, 80-wide grids): the CTA's 64 x (kh + kw) table rows are staged in shared memory once,
    // so the per-score bias is two LDS instead of two scattered global loads
    const int rel_ld = p.kh + p.kw + 1;
    float* rel_s = reinterpret_cast<float*>(smem + 2 * STAGE);
    if (has_rel && !hoist) {
        for (int i = threadIdx.x; i < ATT_BM * (p.kh + p.kw); i += 128) {
            const int rr = i / (p.kh + p.kw), c = i - rr * (p.kh + p.kw);
            const int qq = min(q0 + rr, p.Tq - 1);
            const int64_t rowi = ((int64_t)b * p.H + h) * p.Tq + qq;
            rel_s[rr * rel_ld + c] = c < p.kh ? __ldg(p.rel_h + rowi * p.kh + c) : __ldg(p.rel_w + rowi * p.kw + (c - p.kh));
        }
        __syncthreads();
    }
    const float* rs0 = rel_s + (warp * 16 + (lane >> 2)) * rel_ld;
    const float* rs1 = rs0 + 8 * rel_ld;
    float rw[ATT_BN / 8][4];
    if (hoist) {
#pragma unroll
        for (int j = 0; j < ATT_BN / 8; ++j) {
            const float2 a = *reinterpret_cast<const float2*>(relw_r[0] + j * 8 + (lane & 3) * 2);
            const float2 c = *reinterpret_cast<const float2*>(relw_r[1] + j * 8 + (lane & 3) * 2);
            rw[j][0] = a.x; rw[j][1] = a.y; rw[j][2] = c.x; rw[j][3] = c.y;
        }
    }
    constexpr float LOG2E = 1.4426950408889634f;

    const int ntiles = (p.Tk + ATT_BN - 1) / ATT_BN;
    for (int t = 0; t < ntiles; ++t) {
        const int kv0 = t * ATT_BN;
        if (t + 1 < ntiles) load_tile((t + 1) & 1, kv0 + ATT_BN);
        cp_async_commit();
        cp_async_wait<1>();
        __syncthreads();
        const uint32_t sb = smem_base + (t & 1) * STAGE;

        // ---- S = Q K^T ----
        float s[ATT_BN / 8][4];
#pragma unroll
        for (int j = 0; j < ATT_BN / 8; ++j) s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
        {
            const int key_l = (lane & 7) + (lane >> 4) * 8;
            const int cb = ((lane >> 3) & 1) * 16;
#pragma unroll
            for (int kk = 0; kk < KSTEPS; ++kk) {
#pragma unroll
                for (int j = 0; j < ATT_BN / 8; j += 2) {
                    uint32_t b0, b1, b2, b3;
                    ldsm_x4(sb + (j * 8 + key_l) * ROWB + kk * 32 + cb, b0, b1, b2, b3);
                    mma_bf16(s[j], qa_hi[kk], b0, b1);
                    mma_bf16(s[j + 1], qa_hi[kk], b2, b3);
                    if (PREC == 3) {
                        mma_bf16(s[j], qa_lo[kk], b0, b1);
                        mma_bf16(s[j + 1], qa_lo[kk], b2, b3);
                        uint32_t c0, c1, c2, c3;
                        ldsm_x4(sb + PLANE + (j * 8 + key_l) * ROWB + kk * 32 + cb, c0, c1, c2, c3);
                        mma_bf16(s[j], qa_hi[kk], c0, c1);
                        mma_bf16(s[j + 1], qa_hi[kk], c2, c3);
                    }
                }
            }
        }
        // ---- scale + bias + mask, online softmax ----
        float mx[2] = {-INFINITY, -INFINITY};
        float rh0 = 0.f, rh1 = 0.f;
        if (hoist) { rh0 = __ldg(relh_r[0] + t); rh1 = __ldg(relh_r[1] + t); }
        uint32_t km0[2] = {0u, 0u}, km1[2] = {0u, 0u};       // mask words of this 64-key tile
        if (km_r[0]) {
#pragma unroll
            for (int w = 0; w < 2; ++w) {
                const int wi = t * 2 + w;
                km0[w] = wi < mask_words ? __ldg(km_r[0] + wi) : 0u;
                km1[w] = wi < mask_words ? __ldg(km_r[1] + wi) : 0u;
            }
        }
#pragma unroll
        for (int j = 0; j < ATT_BN / 8; ++j) {
            const int key = kv0 + j * 8 + (lane & 3) * 2;
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int kk = key + e;
                const bool ok = kk < p.Tk;
                float add0 = 0.f, add1 = 0.f;
                if (ok) {
                    if (hoist) {
                        add0 = rh0 + rw[j][e];
                        add1 = rh1 + rw[j][2 + e];
                    } else if (has_rel) {
                        const int khi = kk / p.kw, kwi = kk - khi * p.kw;
                        add0 = rs0[khi] + rs0[p.kh + kwi];
                        add1 = rs1[khi] + rs1[p.kh + kwi];
                    }
                    if (kb) { const float kbv = __ldg(kb + kk); add0 += kbv; add1 += kbv; }
                }
                const int kbit = (j * 8 + (lane & 3) * 2 + e) & 31, kw_ = j >> 2;       // key index inside the tile: word j / 4
                const bool ok0 = ok && !((km0[kw_] >> kbit) & 1u), ok1 = ok && !((km1[kw_] >> kbit) & 1u);
                s[j][e] = ok0 ? s[j][e] * p.scale + add0 : -INFINITY;
                s[j][2 + e] = ok1 ? s[j][2 + e] * p.scale + add1 : -INFINITY;
                mx[0] = fmaxf(mx[0], s[j][e]);
                mx[1] = fmaxf(mx[1], s[j][2 + e]);
            }
        }
        float corr[2], msafe[2];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            mx[i] = fmaxf(mx[i], __shfl_xor_sync(0xffffffffu, mx[i], 1));
            mx[i] = fmaxf(mx[i], __shfl_xor_sync(0xffffffffu, mx[i], 2));
            const float mnew = fmaxf(m_run[i], mx[i]);
            msafe[i] = mnew == -INFINITY ? 0.f : mnew;
            corr[i] = ex2_approx((m_run[i] - msafe[i]) * LOG2E);  // m_run = -inf -> 0
            m_run[i] = mnew;
            l_run[i] *= corr[i];
        }
#pragma unroll
        for (int j = 0; j < DTILES; ++j) {
            o[j][0] *= corr[0]; o[j][1] *= corr[0];
            o[j][2] *= corr[1]; o[j][3] *= corr[1];
        }
        uint32_t pa_hi[ATT_BN / 16][4], pa_lo[PREC == 3 ? ATT_BN / 16 : 1][4];
#pragma unroll
        for (int j = 0; j < ATT_BN / 8; ++j) {
            const float p0 = ex2_approx((s[j][0] - msafe[0]) * LOG2E), p1 = ex2_approx((s[j][1] - msafe[0]) * LOG2E);
            const float p2 = ex2_approx((s[j][2] - msafe[1]) * LOG2E), p3 = ex2_approx((s[j][3] - msafe[1]) * LOG2E);
            l_run[0] += p0 + p1;
            l_run[1] += p2 + p3;
            const int kk = j >> 1, half = (j & 1) * 2;
            if (PREC == 3) {
                split2(p0, p1, pa_hi[kk][half], pa_lo[kk][half]);
                split2(p2, p3, pa_hi[kk][half + 1], pa_lo[kk][half + 1]);
            } else {
                pa_hi[kk][half] = pack_bf16x2(p0, p1);
                pa_hi[kk][half + 1] = pack_bf16x2(p2, p3);
            }
        }
        // ---- O += P V ----
        {
            const int key_l = (lane & 7) + ((lane >> 3) & 1) * 8;
            const int cb = (lane >> 4) * 16;
#pragma unroll
            for (int kk = 0; kk < ATT_BN / 16; ++kk) {
#pragma unroll
                for (int j = 0; j < DTILES; j += 2) {
                    uint32_t b0, b1, b2, b3;
                    ldsm_x4_t(sb + VPL * PLANE + (kk * 16 + key_l) * ROWB + j * 16 + cb, b0, b1, b2, b3);
                    mma_bf16(o[j], pa_hi[kk], b0, b1);
                    mma_bf16(o[j + 1], pa_hi[kk], b2, b3);
                    if (PREC == 3) {
                        mma_bf16(o[j], pa_lo[kk], b0, b1);
                        mma_bf16(o[j + 1], pa_lo[kk], b2, b3);
                        uint32_t c0, c1, c2, c3;
                        ldsm_x4_t(sb + (VPL + 1) * PLANE + (kk * 16 + key_l) * ROWB + j * 16 + cb, c0, c1, c2, c3);
                        mma_bf16(o[j], pa_hi[kk], c0, c1);
                        mma_bf16(o[j + 1], pa_hi[kk], c2, c3);
                    }
                }
            }
        }
        __syncthreads();  // everyone done with this stage before it is refilled
    }
    cp_async_wait<0>();

    // ---- finalise ----
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        l_run[i] += __shfl_xor_sync(0xffffffffu, l_run[i], 1);
        l_run[i] += __shfl_xor_sync(0xffffffffu, l_run[i], 2);
    }
    const float inv[2] = {l_run[0] > 0.f ? 1.f / l_run[0] : 0.f, l_run[1] > 0.f ? 1.f / l_run[1] : 0.f};
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        if (qrow[i] >= p.Tq) continue;
        const int64_t base = (int64_t)b * p.o_bs + (int64_t)qrow[i] * p.o_ts + (int64_t)h * HD + (lane & 3) * 2;
#pragma unroll
        for (int j = 0; j < DTILES; ++j) {
            const float a = o[j][2 * i] * inv[i], c = o[j][2 * i + 1] * inv[i];
            if (p.out_f32) *reinterpret_cast<float2*>(p.out_f32 + base + j * 8) = make_float2(a, c);
            if (p.out_hi) {
                uint32_t hi, lo;
                split2(a, c, hi, lo);
                *reinterpret_cast<uint32_t*>(p.out_hi + base + j * 8) = hi;
                if (p.out_lo) *reinterpret_cast<uint32_t*>(p.out_lo + base + j * 8) = lo;
            }
        }
    }
}

// rel[b,h,q,j] = sum_c q[b,q,h,c] * Rt[coord(q)][c][j]   (Rt pre-transposed: (qsize, hd, ksize))
// one warp per (b, h, q); lanes over j.
__global__ void __launch_bounds__(256)
relpos_kernel(const __nv_bfloat16* __restrict__ q_hi, const __nv_bfloat16* __restrict__ q_lo, int64_t q_bs,
              int64_t q_ts, int64_t q_hs, const float* __restrict__ Rt, int axis, int qh, int qw, int ksize,
              float* __restrict__ rel, int B, int H, int hd) {
    const int lane = threadIdx.x & 31;
    const int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int T = qh * qw;
    if (w >= (int64_t)B * H * T) return;
    const int q = (int)(w % T);
    const int h = (int)((w / T) % H);
    const int b = (int)(w / ((int64_t)T * H));
    const int coord = axis == 0 ? q / qw : q % qw;
    const __nv_bfloat16* qp = q_hi + (int64_t)b * q_bs + (int64_t)q * q_ts + (int64_t)h * q_hs;
    const __nv_bfloat16* ql = q_lo ? q_lo + (int64_t)b * q_bs + (int64_t)q * q_ts + (int64_t)h * q_hs : nullptr;
    // lane c holds q[c], q[c+32], q[c+64], q[c+96]
    float qv[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int c = lane + 32 * i;
        qv[i] = c < hd ? __bfloat162float(qp[c]) + (ql ? __bfloat162float(ql[c]) : 0.f) : 0.f;
    }
    const float* Rb = Rt + (int64_t)coord * hd * ksize;
    for (int j0 = 0; j0 < ksize; j0 += 32) {
        const int j = j0 + lane;
        float acc = 0.f;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int cmax = min(32, hd - 32 * i);
            for (int cc = 0; cc < cmax; ++cc) {
                const float qc = __shfl_sync(0xffffffffu, qv[i], cc);
                if (j < ksize) acc += qc * __ldg(Rb + (int64_t)(32 * i + cc) * ksize + j);
            }
        }
        if (j < ksize) rel[w * ksize + j] = acc;
    }
}


// ------------------------------------------------------------------------------------------
// Decomposed rel-pos tables on tensor cores.  Queries that share a grid coordinate (same row for the
// height axis, same column for the width axis) share the (ksize x hd) table R[coord], so
//   rel[b,h,q,:] = q[b,q,h,:] . R[coord(q)]^T
// is a (G x hd) x (hd x ksize) GEMM per (b, h, coord) group of G queries.  One CTA = one (coord, b, h)
// group; R[coord] (bf16 hi/lo, K-major) is staged in shared memory, each warp computes m16 slabs with
// mma.sync in bf16x3 (fp32-class) and stores fp32.
// ------------------------------------------------------------------------------------------
// F16: q is one IEEE fp16 plane and the table planes are fp16 hi/lo (q.Rh + q.Rl): the companion of the single-pass fp16 attention.
template <int HD, bool F16>
__global__ void __launch_bounds__(128)
relpos_mma_kernel(const __nv_bfloat16* __restrict__ q_hi, const __nv_bfloat16* __restrict__ q_lo, int64_t q_bs,
                  int64_t q_ts, int64_t q_hs, const __nv_bfloat16* __restrict__ R_hi,
                  const __nv_bfloat16* __restrict__ R_lo, int axis, int qh, int qw, int ksize, int kpad,
                  float* __restrict__ rel, int B, int H) {
    constexpr int ROWB = HD * 2 + 16;
    constexpr int KSTEPS = HD / 16;
    constexpr int CHUNKS = HD / 8;
    extern __shared__ __align__(16) uint8_t smem[];
    const uint32_t sb = (uint32_t)__cvta_generic_to_shared(smem);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int coord = blockIdx.x, b = blockIdx.z;            // one CTA per (coordinate, batch): R[coord] is staged once for all heads
    const int G = axis == 0 ? qw : qh;                       // queries sharing this coordinate
    const int T = qh * qw;
    // stage R[coord] (kpad rows x HD), rows >= ksize zero-filled
    for (int pl = 0; pl < 2; ++pl) {
        const __nv_bfloat16* src = (pl == 0 ? R_hi : R_lo) + (int64_t)coord * ksize * HD;
        for (int i = threadIdx.x; i < kpad * CHUNKS; i += 128) {
            const int r = i / CHUNKS, c = i - r * CHUNKS;
            const bool ok = r < ksize;
            cp_async16(sb + pl * kpad * ROWB + r * ROWB + c * 16, src + (int64_t)(ok ? r : 0) * HD + c * 8, ok ? 16 : 0);
        }
    }
    cp_async_commit();
    cp_async_wait<0>();
    __syncthreads();
    const int nslabs = (G + 15) / 16;
    const int hpc = (H + gridDim.y - 1) / gridDim.y;         // heads per CTA
    for (int wk = warp; wk < hpc * nslabs; wk += 4) {
        const int h = blockIdx.y * hpc + wk / nslabs, slab = wk % nslabs;
        if (h >= H) break;
        // the slab's 16 query rows (members g of the group) -> this warp's smem region in 16-byte chunks (whole 160-byte rows,
        // full sectors), then A fragments with ldmatrix
        const int g0 = slab * 16 + (lane >> 2), g1 = g0 + 8;
        auto tok = [&](int g) { return axis == 0 ? coord * qw + g : g * qw + coord; };
        const bool ok0 = g0 < G, ok1 = g1 < G;
        const uint32_t qs = sb + 2 * kpad * ROWB + warp * (2 * 16 * ROWB);
        __syncwarp();                                            // previous work item's ldmatrix reads are done
        for (int i = lane; i < 2 * 16 * CHUNKS; i += 32) {
            const int pl = i / (16 * CHUNKS), rc = i - pl * (16 * CHUNKS);
            const int r = rc / CHUNKS, c = rc - r * CHUNKS;
            const int g = slab * 16 + r;
            const bool ok = g < G && (pl == 0 || q_lo != nullptr);
            const __nv_bfloat16* src = (pl == 0 ? q_hi : (q_lo ? q_lo : q_hi)) + (int64_t)b * q_bs + (int64_t)tok(ok ? g : 0) * q_ts +
                                       (int64_t)h * q_hs + c * 8;
            cp_async16(qs + pl * 16 * ROWB + r * ROWB + c * 16, src, ok ? 16 : 0);
        }
        cp_async_commit();
        cp_async_wait<0>();
        __syncwarp();
        uint32_t ah[KSTEPS][4], al[KSTEPS][4];
        {
            const uint32_t arow = qs + (lane & 15) * ROWB + (lane >> 4) * 16;
#pragma unroll
            for (int kk = 0; kk < KSTEPS; ++kk) {
                ldsm_x4(arow + kk * 32, ah[kk][0], ah[kk][1], ah[kk][2], ah[kk][3]);
                if (q_lo) ldsm_x4(arow + 16 * ROWB + kk * 32, al[kk][0], al[kk][1], al[kk][2], al[kk][3]);
            }
        }
        const int key_l = (lane & 7) + (lane >> 4) * 8;
        const int cb = ((lane >> 3) & 1) * 16;
        for (int j = 0; j < kpad / 8; j += 2) {
            float c0[4] = {0.f, 0.f, 0.f, 0.f}, c1[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int kk = 0; kk < KSTEPS; ++kk) {
                uint32_t b0, b1, b2, b3;
                ldsm_x4(sb + (j * 8 + key_l) * ROWB + kk * 32 + cb, b0, b1, b2, b3);
                mma_16b<F16>(c0, ah[kk], b0, b1);
                mma_16b<F16>(c1, ah[kk], b2, b3);
                if (q_lo) {
                    mma_16b<F16>(c0, al[kk], b0, b1);
                    mma_16b<F16>(c1, al[kk], b2, b3);
                }
                uint32_t d0, d1, d2, d3;
                ldsm_x4(sb + kpad * ROWB + (j * 8 + key_l) * ROWB + kk * 32 + cb, d0, d1, d2, d3);
                mma_16b<F16>(c0, ah[kk], d0, d1);
                mma_16b<F16>(c1, ah[kk], d2, d3);
            }
            const int col = j * 8 + (lane & 3) * 2;
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                const float* c = half == 0 ? c0 : c1;
                const int cc = col + half * 8;
                const bool pair_ok = cc + 1 < ksize && (ksize & 1) == 0;     // 8-byte aligned pair -> one store
                if (ok0) {
                    float* o = rel + ((((int64_t)b * H + h) * T) + tok(g0)) * ksize + cc;
                    if (pair_ok) *reinterpret_cast<float2*>(o) = make_float2(c[0], c[1]);
                    else {
                        if (cc < ksize) o[0] = c[0];
                        if (cc + 1 < ksize) o[1] = c[1];
                    }
                }
                if (ok1) {
                    float* o = rel + ((((int64_t)b * H + h) * T) + tok(g1)) * ksize + cc;
                    if (pair_ok) *reinterpret_cast<float2*>(o) = make_float2(c[2], c[3]);
                    else {
                        if (cc < ksize) o[0] = c[2];
                        if (cc + 1 < ksize) o[1] = c[3];
                    }
                }
            }
        }
    }
}

template <int HD, int PREC>
static int launch_attn(const AttnParams& p, cudaStream_t st) {
    constexpr int ROWB = HD * 2 + 16;
    constexpr int SMEM_KV = 2 * (PREC == 3 ? 4 : 2) * ATT_BN * ROWB;
    const bool tables = p.rel_h != nullptr && p.kw != ATT_BN;
    const int SMEM = SMEM_KV + (tables ? ATT_BM * (p.kh + p.kw + 1) * (int)sizeof(float) : 0);
    HIPIE_CHECK_ARG(SMEM <= 200 * 1024, "hipie_attention: rel-pos grid %dx%d too large for the shared-memory tables", p.kh, p.kw);
    HIPIE_ENSURE_SMEM((attention_kernel<HD, PREC>), SMEM);
    dim3 grid((p.Tq + ATT_BM - 1) / ATT_BM, p.H, p.B);
    attention_kernel<HD, PREC><<<grid, 128, SMEM, st>>>(p);
    HIPIE_CHECK_LAUNCH();
    return HIPIE_OK;
}

}  // namespace hipie

using namespace hipie;

extern "C" int hipie_attention(const hipie_attn_args* a, void* stream) {
    HIPIE_CHECK_ARG(a, "hipie_attention: null args");
    HIPIE_CHECK_ARG(a->q_hi && a->k_hi && a->v_hi, "hipie_attention: q/k/v hi planes required");
    HIPIE_CHECK_ARG(a->prec == 1 || (a->prec == 3 && a->q_lo && a->k_lo && a->v_lo), "hipie_attention: prec/lo planes mismatch");
    HIPIE_CHECK_ARG(a->out_f32 || a->out_hi, "hipie_attention: no output requested");
    HIPIE_CHECK_ARG(a->B > 0 && a->H > 0 && a->Tq > 0 && a->Tk > 0, "hipie_attention: bad sizes");
    HIPIE_CHECK_ARG((a->rel_h == nullptr) == (a->rel_w == nullptr), "hipie_attention: rel_h and rel_w go together");
    HIPIE_CHECK_ARG(!a->rel_h || (a->kh > 0 && a->kw > 0 && a->kh * a->kw == a->Tk), "hipie_attention: kh*kw must equal Tk");
    HIPIE_CHECK_ARG(a->q_ts % 8 == 0 && a->k_ts % 8 == 0 && a->v_ts % 8 == 0 && a->q_hs % 8 == 0 && a->k_hs % 8 == 0 &&
                        a->v_hs % 8 == 0 && a->q_bs % 8 == 0 && a->k_bs % 8 == 0 && a->v_bs % 8 == 0,
                    "hipie_attention: strides must be multiples of 8 elements (16 bytes)");
    AttnParams p;
    p.q_hi = (const __nv_bfloat16*)a->q_hi; p.q_lo = (const __nv_bfloat16*)a->q_lo;
    p.k_hi = (const __nv_bfloat16*)a->k_hi; p.k_lo = (const __nv_bfloat16*)a->k_lo;
    p.v_hi = (const __nv_bfloat16*)a->v_hi; p.v_lo = (const __nv_bfloat16*)a->v_lo;
    p.q_bs = a->q_bs; p.q_ts = a->q_ts; p.q_hs = a->q_hs;
    p.k_bs = a->k_bs; p.k_ts = a->k_ts; p.k_hs = a->k_hs;
    p.v_bs = a->v_bs; p.v_ts = a->v_ts; p.v_hs = a->v_hs;
    p.rel_h = a->rel_h; p.rel_w = a->rel_w; p.kh = a->kh; p.kw = a->kw;
    p.key_bias = a->key_bias;
    p.key_mask = a->key_mask;
    p.out_f32 = a->out_f32; p.out_hi = (__nv_bfloat16*)a->out_hi; p.out_lo = (__nv_bfloat16*)a->out_lo;
    p.o_bs = a->o_bs; p.o_ts = a->o_ts;
    p.B = a->B; p.H = a->H; p.Tq = a->Tq; p.Tk = a->Tk; p.scale = a->scale;
    cudaStream_t st = (cudaStream_t)stream;
#define HIPIE_ATT(HDV)                                                              \
    if (a->hd == HDV) return a->prec == 3 ? launch_attn<HDV, 3>(p, st) : launch_attn<HDV, 1>(p, st)
    HIPIE_ATT(32);
    HIPIE_ATT(64);
    HIPIE_ATT(80);
#undef HIPIE_ATT
    set_error("hipie_attention: unsupported head dim %d (supported: 32, 64, 80)", a->hd);
    return HIPIE_EUNSUPPORTED;
}

extern "C" int hipie_relpos_bias(const void* q_hi, const void* q_lo, int64_t q_bs, int64_t q_ts, int64_t q_hs,
                                 const float* table_t, int axis, int qh, int qw, int ksize, float* rel, int B, int H,
                                 int hd, void* stream) {
    HIPIE_CHECK_ARG(q_hi && table_t && rel, "hipie_relpos_bias: null pointer");
    HIPIE_CHECK_ARG(hd <= 128 && (axis == 0 || axis == 1), "hipie_relpos_bias: hd <= 128, axis in {0,1}");
    const int64_t warps = (int64_t)B * H * qh * qw;
    if (warps == 0) return HIPIE_OK;
    relpos_kernel<<<(unsigned)((warps + 7) / 8), 256, 0, (cudaStream_t)stream>>>(
        (const __nv_bfloat16*)q_hi, (const __nv_bfloat16*)q_lo, q_bs, q_ts, q_hs, table_t, axis, qh, qw, ksize, rel, B, H, hd);
    HIPIE_CHECK_LAUNCH();
    return HIPIE_OK;
}


// table given as bf16 hi/lo planes of get_rel_pos output, (qsize, ksize, hd) K-major (no transpose needed)
extern "C" int hipie_relpos_bias_tc(const void* q_hi, const void* q_lo, int64_t q_bs, int64_t q_ts, int64_t q_hs,
                                    const void* table_hi, const void* table_lo, int axis, int qh, int qw, int ksize,
                                    float* rel, int B, int H, int hd, void* stream) {
    HIPIE_CHECK_ARG(q_hi && table_hi && table_lo && rel, "hipie_relpos_bias_tc: null pointer");
    HIPIE_CHECK_ARG(axis == 0 || axis == 1, "hipie_relpos_bias_tc: axis in {0,1}");
    HIPIE_CHECK_ARG(q_ts % 8 == 0 && q_hs % 8 == 0 && q_bs % 8 == 0 && ((reinterpret_cast<uintptr_t>(q_hi) | reinterpret_cast<uintptr_t>(q_lo)) & 15) == 0,
                    "hipie_relpos_bias_tc: q rows must be 16-byte aligned (strides multiples of 8 elements)");
    if ((int64_t)B * H * qh * qw == 0) return HIPIE_OK;
    const int kpad = (ksize + 15) / 16 * 16;
    // R[coord] is staged once per CTA and reused for several heads: all heads for short groups (windows: one 16-row slab per
    // head), 4 heads per CTA for the 64-query groups of the global grid (keeps ~2000 CTAs in flight)
    const int G = axis == 0 ? qw : qh;
    const int hpc = G >= 32 ? 4 : 16;
    dim3 grid(axis == 0 ? qh : qw, (H + hpc - 1) / hpc, B);
    cudaStream_t st = (cudaStream_t)stream;
#define HIPIE_RP(HDV)                                                                                           \
    if (hd == HDV) {                                                                                            \
        const int smem = (2 * kpad + 4 * 2 * 16) * (HDV * 2 + 16);       /* R[coord] planes + per-warp Q slabs */ \
        HIPIE_ENSURE_SMEM((relpos_mma_kernel<HDV, false>), smem);                                               \
        relpos_mma_kernel<HDV, false><<<grid, 128, smem, st>>>((const __nv_bfloat16*)q_hi, (const __nv_bfloat16*)q_lo, q_bs, q_ts, \
                                                         q_hs, (const __nv_bfloat16*)table_hi,                  \
                                                         (const __nv_bfloat16*)table_lo, axis, qh, qw, ksize, kpad, rel, B, H); \
        HIPIE_CHECK_LAUNCH();                                                                                   \
        return HIPIE_OK;                                                                                        \
    }
    HIPIE_RP(32)
    HIPIE_RP(64)
    HIPIE_RP(80)
#undef HIPIE_RP
    set_error("hipie_relpos_bias_tc: unsupported head dim %d", hd);
    return HIPIE_EUNSUPPORTED;
}


extern "C" int hipie_relpos_bias_tc_f16(const void* q_f16, int64_t q_bs, int64_t q_ts, int64_t q_hs, const void* table_hi,
                                        const void* table_lo, int axis, int qh, int qw, int ksize, float* rel, int B, int H, int hd,
                                        void* stream) {
    HIPIE_CHECK_ARG(q_f16 && table_hi && table_lo && rel, "hipie_relpos_bias_tc_f16: null pointer");
    HIPIE_CHECK_ARG(axis == 0 || axis == 1, "hipie_relpos_bias_tc_f16: axis in {0,1}");
    HIPIE_CHECK_ARG(q_ts % 8 == 0 && q_hs % 8 == 0 && q_bs % 8 == 0 && (reinterpret_cast<uintptr_t>(q_f16) & 15) == 0,
                    "hipie_relpos_bias_tc_f16: q rows must be 16-byte aligned (strides multiples of 8 elements)");
    if ((int64_t)B * H * qh * qw == 0) return HIPIE_OK;
    const int kpad = (ksize + 15) / 16 * 16;
    const int G = axis == 0 ? qw : qh;
    const int hpc = G >= 32 ? 4 : 16;
    dim3 grid(axis == 0 ? qh : qw, (H + hpc - 1) / hpc, B);
    cudaStream_t st = (cudaStream_t)stream;
#define HIPIE_RPF(HDV)                                                                                          \
    if (hd == HDV) {                                                                                            \
        const int smem = (2 * kpad + 4 * 2 * 16) * (HDV * 2 + 16);                                              \
        HIPIE_ENSURE_SMEM((relpos_mma_kernel<HDV, true>), smem);                                                \
        relpos_mma_kernel<HDV, true><<<grid, 128, smem, st>>>((const __nv_bfloat16*)q_f16, nullptr, q_bs, q_ts, q_hs,       \
                                                              (const __nv_bfloat16*)table_hi, (const __nv_bfloat16*)table_lo, axis, qh, \
                                                              qw, ksize, kpad, rel, B, H);                        \
        HIPIE_CHECK_LAUNCH();                                                                                   \
        return HIPIE_OK;                                                                                        \
    }
    HIPIE_RPF(32)
    HIPIE_RPF(64)
    HIPIE_RPF(80)
#undef HIPIE_RPF
    set_error("hipie_relpos_bias_tc_f16: unsupported head dim %d", hd);
    return HIPIE_EUNSUPPORTED;
}
