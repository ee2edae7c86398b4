// wgmma flash attention for the ViT-H blocks (hd = 80), sm_90a (H100): global 64-wide token grids (T % 256 == 0), 80-wide ones
// (1280-pixel inputs; T % 1280 == 0) and the 14x14 windows.
//
//   softmax((q*scale) k^T + rel_h[q, kh] + rel_w[q, kw]) v      (reference hipie/backbone/vit.py:67-83, backbone/utils.py:96-125)
//
// One CTA = 128 query rows of one (batch, head); 384 threads in three warpgroups:
//   warpgroup 0     TMA producer (one thread): the Q tiles once, then K tiles (64 keys x 80) and V^T tiles (80 x 64 keys) into a
//                   3-stage hardware-swizzled shared-memory ring (head dim 80 = one 128B-swizzled 64-wide box + one 32B-swizzled
//                   16-wide box)
//   warpgroups 1-2  64 query rows each: S = Q K^T (wgmma m64n64k16, both operands in shared memory), scale + rel-pos bias and the
//                   online softmax on the register fragment, P packed in registers as the A operand of O += P V (wgmma m64n80k16,
//                   A from registers), O in registers; S(j+1) is issued before the softmax of tile j, and the two warpgroups take
//                   turns on the tensor cores (schedule at the key loop)
//   window mode (T = 196, 14 x 14): keys padded to 4 x 64 and masked; V^T holds every window at a 200-column pitch because TMA
//                   box starts must be 16-byte aligned
// Precision: PREC==3 evaluates Qh.Kh + Qh.Kl + Ql.Kh and Ph.Vh + Ph.Vl + Pl.Vh (bf16x3, fp32-class); PREC==1 plain bf16 (or fp16).
#include "common.cuh"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace hipie {
using namespace ptx;

int make_tmap_bf16(CUtensorMap* out, const void* ptr, int64_t rows, int64_t cols, int64_t ld, int batch,
                   int64_t bstride, int box_rows, int box_cols);

constexpr int FA_BM = 64, FA_BN = 64, FA_HD = 80, FA_STAGES = 3;
constexpr int FA_CONSUMERS = 2;                        // consumer warpgroups per CTA, FA_BM query rows each
constexpr int FA_THREADS = 128 * (1 + FA_CONSUMERS);   // + the producer warpgroup (one TMA thread)
// setmaxnreg split of the 168 registers per thread of a 384-thread CTA: 24 + 2 x 240 = 3 x 168
constexpr int FA_PRODUCER_REGS = 24, FA_CONSUMER_REGS = 240;
constexpr int FA_BAR_TURN = 3;                         // named barriers 3, 4: tensor-core turn of consumer 0, 1 (1, 2: epilogue)
constexpr int FA_OLD = FA_HD + 4;                      // row length (floats) of the staged output tile

struct FaMaps {
    CUtensorMap k64[2], k16[2], vt[2];   // [hi, lo]
    CUtensorMap q64[2], q16[2];
};

struct FaParams {
    const float *rel_h, *rel_w;   // (B,H,T,kh), (B,H,T,kw) or null
    int kh;
    float* out_f32;
    __nv_bfloat16 *out_hi, *out_lo;
    int out_e4m3;        // out_hi is ONE fp16 plane, out_lo the e4m3 planes (B*T rows of 2*o_ts bytes): the A operand of a prec-6 proj GEMM
    int64_t o_bs, o_ts;
    int B, H, T;
    int T_rows;          // rows per batch item of the output (o_bs / o_ts)
    int q_col0, k_col0;           // column of head 0 inside the q / k rows
    float scale_log2e;
};

template <int PREC>
struct FaSmem {
    static constexpr int NPL = PREC == 3 ? 2 : 1;
    static constexpr int K64 = FA_BN * 128, K16 = FA_BN * 32;
    static constexpr int VT = FA_HD * 128;
    static constexpr int K_STAGE = NPL * (K64 + K16);
    static constexpr int V_STAGE = NPL * VT;
    static constexpr int Q64 = FA_BM * 128, Q16 = FA_BM * 32;
    static constexpr int Q_TILE = NPL * (Q64 + Q16);
    static constexpr int OFF_V = FA_STAGES * K_STAGE;
    static constexpr int OFF_Q = OFF_V + FA_STAGES * V_STAGE;
    static constexpr int OFF_O = OFF_Q + FA_CONSUMERS * Q_TILE;
    static constexpr int OFF_BAR = OFF_O + FA_CONSUMERS * FA_BM * FA_OLD * 4;
    static constexpr int TOTAL = OFF_BAR + 256 + 1024;
};

constexpr int FA_GW2 = 80;        // second supported global grid width (1280-pixel inputs)
constexpr int FA_WIN = 14, FA_WIN_T = FA_WIN * FA_WIN;     // window mode: 14 x 14 tokens, keys padded to 4 x 64
constexpr int FA_WIN_TP = 200;   // window mode: column pitch of one window in V^T (TMA box starts must be 16-byte aligned)

// S (+)= Q . K^T over the head dim 80: one 128B-swizzled 64-wide box (4 wgmmas) + one 32B-swizzled 16-wide box
template <bool F16>
__device__ __forceinline__ void fa_qk(float (&sacc)[32], uint32_t q, uint32_t k, int qoff16, int koff16, bool first) {
    const uint64_t q64 = wg::desc<128>(q), q16 = wg::desc<32>(q + qoff16), k64 = wg::desc<128>(k), k16 = wg::desc<32>(k + koff16);
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
        if (F16) wg::ss_f16_n64(sacc, q64 + 2 * kk, k64 + 2 * kk, !(first && kk == 0));
        else wg::ss_bf16_n64(sacc, q64 + 2 * kk, k64 + 2 * kk, !(first && kk == 0));
    }
    if (F16) wg::ss_f16_n64(sacc, q16, k16, 1);
    else wg::ss_bf16_n64(sacc, q16, k16, 1);
}

template <bool F16>
__device__ __forceinline__ void fa_pv(float (&o)[40], const uint32_t (&pa)[4][4], uint32_t v) {
    const uint64_t dv = wg::desc<128>(v);
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
        if (F16) wg::rs_f16_n80(o, pa[kk], dv + 2 * kk, 1);
        else wg::rs_bf16_n80(o, pa[kk], dv + 2 * kk, 1);
    }
}

// F16 (with PREC == 1): q, k, v^T are IEEE fp16 planes and P is written as fp16: the single-pass QK^T / PV mode of the precision
// map (DESIGN.md 3: 2^-12 operand rounding instead of bf16's 2^-9).
// GW: key-grid width of the rel-pos tables (64 or 80; FA_WIN in window mode).
template <int PREC, bool WIN, bool F16, int GW>
__global__ void __launch_bounds__(FA_THREADS, 1)
attn_tc_kernel(const __grid_constant__ FaMaps maps, const FaParams p) {
    using SM = FaSmem<PREC>;
    constexpr int NPL = SM::NPL;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // stays in the shared address space (LDS / STS)
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + SM::OFF_BAR);
    uint64_t* k_full = bars;                       // [STAGES]
    uint64_t* k_empty = k_full + FA_STAGES;        // [STAGES] one arrival per consumer warp
    uint64_t* v_full = k_empty + FA_STAGES;
    uint64_t* v_empty = v_full + FA_STAGES;
    uint64_t* q_full = v_empty + FA_STAGES;        // [CONSUMERS]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int q0 = blockIdx.x * (FA_CONSUMERS * FA_BM), h = blockIdx.y, b = blockIdx.z;
    const int ntiles = WIN ? (FA_WIN_T + FA_BN - 1) / FA_BN : p.T / FA_BN;     // window mode: 196 keys in 4 tiles, tail masked

    if (threadIdx.x == 0) {
        for (int i = 0; i < NPL; ++i) {
            prefetch_tmap(&maps.k64[i]); prefetch_tmap(&maps.k16[i]); prefetch_tmap(&maps.vt[i]);
            prefetch_tmap(&maps.q64[i]); prefetch_tmap(&maps.q16[i]);
        }
        for (int i = 0; i < FA_STAGES; ++i) {
            mbar_init(&k_full[i], 1); mbar_init(&k_empty[i], 4 * FA_CONSUMERS);
            mbar_init(&v_full[i], 1); mbar_init(&v_empty[i], 4 * FA_CONSUMERS);
        }
        for (int i = 0; i < FA_CONSUMERS; ++i) mbar_init(&q_full[i], 1);
        fence_barrier_init();
    }
    __syncthreads();

    if (warp < 4) {
        // ===================== TMA producer =====================
        setmaxnreg_dec<FA_PRODUCER_REGS>();
        if (threadIdx.x == 0) {
            for (int c = 0; c < FA_CONSUMERS; ++c) {
                uint8_t* qb = smem + SM::OFF_Q + c * SM::Q_TILE;
                mbar_arrive_expect_tx(&q_full[c], SM::Q_TILE);
                for (int pl = 0; pl < NPL; ++pl) {
                    tma_load_3d(qb + pl * (SM::Q64 + SM::Q16), &maps.q64[pl], &q_full[c], p.q_col0 + h * FA_HD, q0 + c * FA_BM, b);
                    tma_load_3d(qb + pl * (SM::Q64 + SM::Q16) + SM::Q64, &maps.q16[pl], &q_full[c], p.q_col0 + h * FA_HD + 64, q0 + c * FA_BM, b);
                }
            }
            int s = 0;
            uint32_t ph = 0;
            for (int j = 0; j < ntiles; ++j) {
                mbar_wait(&k_empty[s], ph ^ 1);
                mbar_arrive_expect_tx(&k_full[s], SM::K_STAGE);
                uint8_t* kb = smem + s * SM::K_STAGE;
                for (int pl = 0; pl < NPL; ++pl) {
                    tma_load_3d(kb + pl * (SM::K64 + SM::K16), &maps.k64[pl], &k_full[s], p.k_col0 + h * FA_HD, j * FA_BN, b);
                    tma_load_3d(kb + pl * (SM::K64 + SM::K16) + SM::K64, &maps.k16[pl], &k_full[s], p.k_col0 + h * FA_HD + 64, j * FA_BN, b);
                }
                mbar_wait(&v_empty[s], ph ^ 1);
                mbar_arrive_expect_tx(&v_full[s], SM::V_STAGE);
                uint8_t* vb = smem + SM::OFF_V + s * SM::V_STAGE;
                for (int pl = 0; pl < NPL; ++pl)
                    tma_load_3d(vb + pl * SM::VT, &maps.vt[pl], &v_full[s], b * (WIN ? FA_WIN_TP : p.T) + j * FA_BN, h * FA_HD, 0);
                if (++s == FA_STAGES) { s = 0; ph ^= 1; }
            }
        }
        return;
    }
    // ===================== consumer warpgroup c: 64 query rows =====================
    setmaxnreg_inc<FA_CONSUMER_REGS>();
    // wgmma fragment: this thread holds rows ra = 16 wq + lane / 4 and ra + 8, columns 8 j + 2 (lane % 4) + {0, 1}
    const int c = (threadIdx.x >> 7) - 1, wq = warp & 3, tig = lane & 3;
    const int ra = 16 * wq + (lane >> 2);
    const int qrow[2] = {q0 + c * FA_BM + ra, q0 + c * FA_BM + ra + 8};
    const bool has_rel = p.rel_h != nullptr;
    // 64-wide grid: key tile j is key row j, so rel_h is one scalar per row and tile, and the key columns of this thread's
    // fragment (rel_w) are the same in every tile. The 80-wide grid and the windows keep one rel_h + rel_w load per score.
    constexpr bool ROW_TILES = !WIN && GW == FA_BN;
    const float* relw_row[2];
    const float* relh_row[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
        const int64_t rowi = ((int64_t)b * p.H + h) * p.T + (qrow[e] < p.T ? qrow[e] : 0);
        relw_row[e] = has_rel ? p.rel_w + rowi * GW : nullptr;
        relh_row[e] = has_rel ? p.rel_h + rowi * (WIN ? FA_WIN : p.kh) : nullptr;
    }
    float rw[2][16];                 // ROW_TILES: rel_w of row e at fragment column x (score index i: x = 2 (i / 4) + i % 2)
    float rh[2] = {0.f, 0.f}, rh_next[2] = {0.f, 0.f};      // ROW_TILES: rel_h of the tile whose scores come next / the one after
    if (ROW_TILES && has_rel) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
#pragma unroll
            for (int x = 0; x < 16; ++x) rw[e][x] = __ldg(relw_row[e] + 8 * (x >> 1) + 2 * tig + (x & 1));
            rh[e] = __ldg(relh_row[e]);
            rh_next[e] = __ldg(relh_row[e] + (ntiles > 1 ? 1 : 0));
        }
    }
    constexpr float LOG2E = 1.4426950408889634f;
    const uint32_t qb = smem_u32(smem + SM::OFF_Q + c * SM::Q_TILE);
    float o[40];
#pragma unroll
    for (int i = 0; i < 40; ++i) o[i] = 0.f;
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};     // running max (log2 domain) / this thread's share of the row sum
    float sacc[32];
    float corr[2];
    uint32_t pa_hi[4][4], pa_lo[4][4];

    // ---- S = Q K^T of tile jt into sacc (PREC 3: Qh.Kh + Qh.Kl + Ql.Kh); the caller commits ----
    auto issue_qk = [&](int jt) {
        const uint32_t kb = smem_u32(smem + (jt % FA_STAGES) * SM::K_STAGE);
        fa_qk<F16>(sacc, qb, kb, SM::Q64, SM::K64, true);
        if (PREC == 3) {
            fa_qk<F16>(sacc, qb, kb + SM::K64 + SM::K16, SM::Q64, SM::K64, false);
            fa_qk<F16>(sacc, qb + SM::Q64 + SM::Q16, kb, SM::Q64, SM::K64, false);
        }
    };
    // ---- O += P V from ring stage s (PREC 3: Ph.Vh + Ph.Vl + Pl.Vh); the caller commits ----
    auto issue_pv = [&](int s) {
        const uint32_t vb = smem_u32(smem + SM::OFF_V + s * SM::V_STAGE);
        fa_pv<F16>(o, pa_hi, vb);
        if (PREC == 3) {
            fa_pv<F16>(o, pa_hi, vb + SM::VT);
            fa_pv<F16>(o, pa_lo, vb);
        }
    };
    // ---- scores of tile jt in the log2 domain, s * scale * log2e + (rel_h[q, key row] + rel_w[q, key column]) * log2e, the
    //      online-softmax update of m and l, and exp2(t - m) in place. O is rescaled by corr later, once its PV has retired. ----
    auto softmax = [&](int jt) {
        float tmax[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int i = 0; i < 32; ++i) {
            const int e = (i >> 1) & 1;
            const int k = jt * FA_BN + 8 * (i >> 2) + 2 * tig + (i & 1);
            float t = sacc[i] * p.scale_log2e;
            if (WIN && k >= FA_WIN_T) t = -INFINITY;
            else if (ROW_TILES && has_rel) t = fmaf(rh[e] + rw[e][2 * (i >> 2) + (i & 1)], LOG2E, t);
            else if (!ROW_TILES && has_rel) t = fmaf(__ldg(relh_row[e] + k / GW) + __ldg(relw_row[e] + k % GW), LOG2E, t);
            sacc[i] = t;
            tmax[e] = fmaxf(tmax[e], t);
        }
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            tmax[e] = fmaxf(tmax[e], __shfl_xor_sync(0xffffffffu, tmax[e], 1));
            tmax[e] = fmaxf(tmax[e], __shfl_xor_sync(0xffffffffu, tmax[e], 2));
            const float mn = fmaxf(m[e], tmax[e]);
            corr[e] = ex2_approx(m[e] - mn);      // m == -inf -> 0
            m[e] = mn;
            l[e] *= corr[e];
        }
#pragma unroll
        for (int i = 0; i < 32; ++i) sacc[i] = ex2_approx(sacc[i] - m[(i >> 1) & 1]);
    };
    // ---- O *= corr, then P packed as the register A operand of the PV wgmma (fragment of S == fragment of A, 16 keys per
    //      k-step). Runs only after the previous PV has retired: it rewrites O and the A registers that PV reads. ----
    auto rescale_pack = [&]() {
#pragma unroll
        for (int i = 0; i < 40; ++i) o[i] *= corr[(i >> 1) & 1];
#pragma unroll
        for (int i = 0; i < 32; i += 2) {
            const int e = (i >> 1) & 1;
            const float e0 = sacc[i], e1 = sacc[i + 1];
            uint32_t hi, lo = 0u;
            if (PREC == 3) {
                split2(e0, e1, hi, lo);
                l[e] += e0 + e1;
            } else if (F16) {
                hi = pack_f16x2(e0, e1);                   // the denominator sums exactly the rounded probabilities the numerator uses
                const float2 r = __half22float2(*reinterpret_cast<const __half2*>(&hi));
                l[e] += r.x + r.y;
            } else {
                hi = pack_bf16x2(e0, e1);
                l[e] += __uint_as_float(hi << 16) + __uint_as_float(hi & 0xffff0000u);
            }
            pa_hi[i >> 3][(i >> 1) & 3] = hi;
            pa_lo[i >> 3][(i >> 1) & 3] = lo;
        }
    };

    // Schedule: iteration j issues S(j+1) = Q K(j+1)^T and O += P(j) V(j) back to back, then computes the softmax of S(j+1)
    // while PV(j) runs. The two warpgroups take turns issuing (named barriers FA_BAR_TURN + c), so that one warpgroup's
    // softmax runs while the other's wgmmas occupy the tensor cores. Warpgroup 0 goes first: warpgroup 1 pre-arrives on its
    // barrier and skips its last arrival, so every barrier phase completes.
    mbar_wait(&q_full[c], 0);
    mbar_wait(&k_full[0], 0);
    wg::fence();
    issue_qk(0);
    wg::commit();
    wg::wait<0>();
    wg::fence_regs(sacc);
    __syncwarp();
    if (lane == 0) mbar_arrive(&k_empty[0]);
    softmax(0);
    rescale_pack();
    if (c == 1) named_bar_arrive(FA_BAR_TURN, 2 * 128);
    // (no wgmma sits under a condition: ptxas serialises every wgmma of the kernel when one does, hence the peeled last tile)
    for (int j = 0; j + 1 < ntiles; ++j) {
        const int s = j % FA_STAGES, s1 = (j + 1) % FA_STAGES;
        if (ROW_TILES && has_rel) {       // one tile ahead: the loads have a whole iteration to land
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                rh[e] = rh_next[e];
                rh_next[e] = __ldg(relh_row[e] + (j + 2 < ntiles ? j + 2 : ntiles - 1));
            }
        }
        mbar_wait(&k_full[s1], ((j + 1) / FA_STAGES) & 1);
        mbar_wait(&v_full[s], (j / FA_STAGES) & 1);
        named_bar_sync(FA_BAR_TURN + c, 2 * 128);
        wg::fence_regs(sacc);
        wg::fence_regs(o);
        wg::fence();
        issue_qk(j + 1);
        wg::commit();
        issue_pv(s);
        wg::commit();
        named_bar_arrive(FA_BAR_TURN + (c ^ 1), 2 * 128);
        wg::wait<1>();                    // S(j+1) retired, PV(j) may still run
        wg::fence_regs(sacc);
        __syncwarp();
        if (lane == 0) mbar_arrive(&k_empty[s1]);
        softmax(j + 1);
        wg::wait<0>();
        wg::fence_regs(o);
        __syncwarp();
        if (lane == 0) mbar_arrive(&v_empty[s]);
        rescale_pack();
    }
    {   // last tile: O += P V
        const int s = (ntiles - 1) % FA_STAGES;
        mbar_wait(&v_full[s], ((ntiles - 1) / FA_STAGES) & 1);
        named_bar_sync(FA_BAR_TURN + c, 2 * 128);
        wg::fence_regs(o);
        wg::fence();
        issue_pv(s);
        wg::commit();
        if (c == 0) named_bar_arrive(FA_BAR_TURN + 1, 2 * 128);
        wg::wait<0>();
        wg::fence_regs(o);
    }
    // ---- epilogue: O / l, staged row-major so that one thread writes 16 consecutive columns of one row ----
    float* os = reinterpret_cast<float*>(smem + SM::OFF_O) + c * FA_BM * FA_OLD;
#pragma unroll
    for (int e = 0; e < 2; ++e) {
        l[e] += __shfl_xor_sync(0xffffffffu, l[e], 1);
        l[e] += __shfl_xor_sync(0xffffffffu, l[e], 2);
        const float inv = 1.f / l[e];
#pragma unroll
        for (int jj = 0; jj < 10; ++jj)
            *reinterpret_cast<float2*>(os + (ra + 8 * e) * FA_OLD + 8 * jj + 2 * tig) = make_float2(o[4 * jj + 2 * e] * inv, o[4 * jj + 2 * e + 1] * inv);
    }
    named_bar_sync(1 + c, 128);
    const int t128 = threadIdx.x & 127;
    const int r = t128 & 63, orow = q0 + c * FA_BM + r;
    if (WIN && orow >= p.T) return;                 // window mode: rows 196..255 are padding
    const int64_t obase = (int64_t)b * p.o_bs + (int64_t)orow * p.o_ts + (int64_t)h * FA_HD;
    for (int cc = (t128 >> 6) * 16; cc < FA_HD; cc += 32) {
        float f[16];
#pragma unroll
        for (int i = 0; i < 16; i += 4) {
            const float4 v = *reinterpret_cast<const float4*>(os + r * FA_OLD + cc + i);
            f[i] = v.x; f[i + 1] = v.y; f[i + 2] = v.z; f[i + 3] = v.w;
        }
        if (p.out_f32) {
#pragma unroll
            for (int i = 0; i < 16; i += 4)
                *reinterpret_cast<float4*>(p.out_f32 + obase + cc + i) = make_float4(f[i], f[i + 1], f[i + 2], f[i + 3]);
        }
        if (p.out_hi && p.out_e4m3) {
            uint4 h0, h1, a8, b8;
            uint2 t;
            split4_f16_e4m3(make_float4(f[0], f[1], f[2], f[3]), t, a8.x, b8.x); h0.x = t.x; h0.y = t.y;
            split4_f16_e4m3(make_float4(f[4], f[5], f[6], f[7]), t, a8.y, b8.y); h0.z = t.x; h0.w = t.y;
            split4_f16_e4m3(make_float4(f[8], f[9], f[10], f[11]), t, a8.z, b8.z); h1.x = t.x; h1.y = t.y;
            split4_f16_e4m3(make_float4(f[12], f[13], f[14], f[15]), t, a8.w, b8.w); h1.z = t.x; h1.w = t.y;
            *reinterpret_cast<uint4*>(p.out_hi + obase + cc) = h0;
            *reinterpret_cast<uint4*>(p.out_hi + obase + cc + 8) = h1;
            uint8_t* o8 = reinterpret_cast<uint8_t*>(p.out_lo) + ((int64_t)b * p.T_rows + orow) * 2 * p.o_ts + e4m3_slot0(h * FA_HD + cc);
            *reinterpret_cast<uint4*>(o8) = a8;              // slot 0 / slot 1 of 16 columns inside one 32-column group (common.cuh)
            *reinterpret_cast<uint4*>(o8 + 32) = b8;
        } else if (p.out_hi) {
            uint4 h0, h1, l0, l1;
            split2(f[0], f[1], h0.x, l0.x); split2(f[2], f[3], h0.y, l0.y);
            split2(f[4], f[5], h0.z, l0.z); split2(f[6], f[7], h0.w, l0.w);
            split2(f[8], f[9], h1.x, l1.x); split2(f[10], f[11], h1.y, l1.y);
            split2(f[12], f[13], h1.z, l1.z); split2(f[14], f[15], h1.w, l1.w);
            *reinterpret_cast<uint4*>(p.out_hi + obase + cc) = h0;
            *reinterpret_cast<uint4*>(p.out_hi + obase + cc + 8) = h1;
            if (p.out_lo) {
                *reinterpret_cast<uint4*>(p.out_lo + obase + cc) = l0;
                *reinterpret_cast<uint4*>(p.out_lo + obase + cc + 8) = l1;
            }
        }
    }
}

template <int PREC, bool WIN, bool F16, int GW = FA_BN>
static int launch_fa(const FaMaps& maps, const FaParams& p, cudaStream_t st) {
    using SM = FaSmem<PREC>;
    HIPIE_ENSURE_SMEM((attn_tc_kernel<PREC, WIN, F16, GW>), SM::TOTAL);
    constexpr int rows = FA_CONSUMERS * FA_BM;
    dim3 grid(((WIN ? FA_WIN_T : p.T) + rows - 1) / rows, p.H, p.B);
    attn_tc_kernel<PREC, WIN, F16, GW><<<grid, FA_THREADS, SM::TOTAL, st>>>(maps, p);
    HIPIE_CHECK_LAUNCH();
    return HIPIE_OK;
}

}  // namespace hipie

using namespace hipie;

static int attention_tc_impl(const void* q_hi, const void* q_lo, int64_t q_bs, int64_t q_ts, int q_col0, int q_width,
                             const void* k_hi, const void* k_lo, int64_t k_bs, int64_t k_ts, int k_col0, int k_width,
                             const void* vt_hi, const void* vt_lo, int64_t vt_ld, const float* rel_h, const float* rel_w,
                             int kh, int kw, float* out_f32, void* out_hi, void* out_lo, int64_t o_bs, int64_t o_ts, int B,
                             int H, int T, int hd, float scale, int prec, void* stream, int out_format) {
    HIPIE_CHECK_ARG(out_format == 0 || (out_format == 1 && out_hi && out_lo && o_ts % 16 == 0 && o_bs % o_ts == 0 && o_ts == (int64_t)H * hd),
                    "hipie_attention_tc: out_format 1 (fp16 + e4m3 planes) needs out_hi, out_lo and contiguous (B, rows, H*hd) outputs");
    HIPIE_CHECK_ARG(q_hi && k_hi && vt_hi, "hipie_attention_tc: q/k/vt hi planes required");
    HIPIE_CHECK_ARG(prec == 1 || prec == 2 || (prec == 3 && q_lo && k_lo && vt_lo), "hipie_attention_tc: prec/lo planes mismatch");
    const bool f16 = prec == 2;          // prec 2: q / k / v^T are single IEEE fp16 planes, one MMA pass
    if (f16) prec = 1;
    HIPIE_CHECK_ARG(hd == FA_HD, "hipie_attention_tc: head dim must be 80 (got %d)", hd);
    const bool win = T == FA_WIN_T && kh == FA_WIN && kw == FA_WIN;      // 14 x 14 windows: one CTA per (window, head)
    HIPIE_CHECK_ARG(win || (T > 0 && T % 256 == 0),
                    "hipie_attention_tc: T (%d) must be a multiple of 256 (or 196 with a 14x14 rel-pos grid: window mode)", T);
    HIPIE_CHECK_ARG((rel_h == nullptr) == (rel_w == nullptr), "hipie_attention_tc: rel_h and rel_w go together");
    const bool wide = !win && rel_h && kw == FA_GW2;       // 80-wide grid: 64-key tiles in 5 phases per 4 key rows
    HIPIE_CHECK_ARG(win || !rel_h || ((kw == FA_BN || (wide && T % (5 * FA_BN) == 0)) && kh * kw == T),
                    "hipie_attention_tc: rel-pos needs a 64-wide grid, or an 80-wide one with T %% 320 == 0, and kh*kw == T");
    HIPIE_CHECK_ARG(out_f32 || out_hi, "hipie_attention_tc: no output requested");
    HIPIE_CHECK_ARG(q_ts % 8 == 0 && q_bs % 8 == 0 && q_col0 % 8 == 0 && (reinterpret_cast<uintptr_t>(q_hi) & 15) == 0,
                    "hipie_attention_tc: q rows must be 16-byte aligned");
    FaMaps maps;
    int rc;
    const void* kp[2] = {k_hi, k_lo};
    const void* vp[2] = {vt_hi, vt_lo};
    for (int pl = 0; pl < (prec == 3 ? 2 : 1); ++pl) {
        if ((rc = make_tmap_bf16(&maps.k64[pl], kp[pl], T, k_width, k_ts, B, k_bs, FA_BN, 64))) return rc;
        if ((rc = make_tmap_bf16(&maps.k16[pl], kp[pl], T, k_width, k_ts, B, k_bs, FA_BN, 16))) return rc;
        if ((rc = make_tmap_bf16(&maps.vt[pl], vp[pl], (int64_t)H * FA_HD, (int64_t)B * (win ? FA_WIN_TP : T), vt_ld, 1, 0, FA_HD, 64))) return rc;
    }
    if (prec == 1) { maps.k64[1] = maps.k64[0]; maps.k16[1] = maps.k16[0]; maps.vt[1] = maps.vt[0]; }
    const void* qp[2] = {q_hi, q_lo};
    for (int pl = 0; pl < (prec == 3 ? 2 : 1); ++pl) {
        if ((rc = make_tmap_bf16(&maps.q64[pl], qp[pl], T, q_width, q_ts, B, q_bs, FA_BM, 64))) return rc;
        if ((rc = make_tmap_bf16(&maps.q16[pl], qp[pl], T, q_width, q_ts, B, q_bs, FA_BM, 16))) return rc;
    }
    if (prec == 1) { maps.q64[1] = maps.q64[0]; maps.q16[1] = maps.q16[0]; }
    FaParams p;
    p.rel_h = rel_h; p.rel_w = rel_w; p.kh = kh;
    p.out_f32 = out_f32; p.out_hi = (__nv_bfloat16*)out_hi; p.out_lo = (__nv_bfloat16*)out_lo;
    p.out_e4m3 = out_format == 1 ? 1 : 0;
    p.T_rows = (int)(o_bs / o_ts);
    p.o_bs = o_bs; p.o_ts = o_ts; p.B = B; p.H = H; p.T = T; p.q_col0 = q_col0; p.k_col0 = k_col0;
    p.scale_log2e = scale * 1.4426950408889634f;
    cudaStream_t st = (cudaStream_t)stream;
    if (wide) return prec == 3 ? launch_fa<3, false, false, FA_GW2>(maps, p, st) : (f16 ? launch_fa<1, false, true, FA_GW2>(maps, p, st) : launch_fa<1, false, false, FA_GW2>(maps, p, st));
    if (win) return prec == 3 ? launch_fa<3, true, false, FA_WIN>(maps, p, st) : (f16 ? launch_fa<1, true, true, FA_WIN>(maps, p, st) : launch_fa<1, true, false, FA_WIN>(maps, p, st));
    return prec == 3 ? launch_fa<3, false, false>(maps, p, st) : (f16 ? launch_fa<1, false, true>(maps, p, st) : launch_fa<1, false, false>(maps, p, st));
}

// Same attention with the output written as the operand planes of a prec-6 hipie_gemm (the proj linear): out_f16 (B, T, H*hd) one
// fp16 plane, out_e4m3 (B*T, 2*H*hd) = [e4m3(h) | e4m3(2^10 (o - h))].
extern "C" int hipie_attention_tc_planes(const void* q_hi, const void* q_lo, int64_t q_bs, int64_t q_ts, int q_col0, int q_width,
                                         const void* k_hi, const void* k_lo, int64_t k_bs, int64_t k_ts, int k_col0, int k_width,
                                         const void* vt_hi, const void* vt_lo, int64_t vt_ld, const float* rel_h, const float* rel_w,
                                         int kh, int kw, float* out_f32, void* out_f16, void* out_e4m3, int64_t o_bs, int64_t o_ts, int B,
                                         int H, int T, int hd, float scale, int prec, void* stream) {
    return attention_tc_impl(q_hi, q_lo, q_bs, q_ts, q_col0, q_width, k_hi, k_lo, k_bs, k_ts, k_col0, k_width, vt_hi, vt_lo, vt_ld, rel_h,
                             rel_w, kh, kw, out_f32, out_f16, out_e4m3, o_bs, o_ts, B, H, T, hd, scale, prec, stream, 1);
}

// Window mode (T == 196, kh == kw == 14): vt holds every window at a 200-column pitch, (H*80, B*200), pad columns zero.
// q / k: bf16 planes viewed as (B, T, row_width) with token stride q_ts / k_ts and batch stride q_bs / k_bs (elements);
// head h occupies columns [q_col0 + 80 h, +80).  vt: V transposed, (H*80 rows, B*T columns) planes with row stride vt_ld.
extern "C" int hipie_attention_tc(const void* q_hi, const void* q_lo, int64_t q_bs, int64_t q_ts, int q_col0, int q_width,
                                  const void* k_hi, const void* k_lo, int64_t k_bs, int64_t k_ts, int k_col0, int k_width,
                                  const void* vt_hi, const void* vt_lo, int64_t vt_ld, const float* rel_h, const float* rel_w,
                                  int kh, int kw, float* out_f32, void* out_hi, void* out_lo, int64_t o_bs, int64_t o_ts, int B,
                                  int H, int T, int hd, float scale, int prec, void* stream) {
    return attention_tc_impl(q_hi, q_lo, q_bs, q_ts, q_col0, q_width, k_hi, k_lo, k_bs, k_ts, k_col0, k_width, vt_hi, vt_lo, vt_ld, rel_h,
                             rel_w, kh, kw, out_f32, out_hi, out_lo, o_bs, o_ts, B, H, T, hd, scale, prec, stream, 0);
}
