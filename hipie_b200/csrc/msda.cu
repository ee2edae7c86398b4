// Multi-scale deformable attention forward for sm_90a.
//
// Semantics follow the reference operator `ms_deform_attn_forward`
// (/root/reference/projects/HIPIE/hipie/models/deformable_detr/ops/src/cuda/ms_deform_attn_cuda.cu:20-78,
//  ms_deform_im2col_cuda.cuh:33-84,237-299) == ms_deform_attn_core_pytorch
// (.../ops/functions/ms_deform_attn_func.py:43-63): pixel = loc * size - 0.5, bilinear with zero
// padding, weighted sum over L levels x P points.  The design is new:
//
//  * fast path (fp32 math, D == 32, L == 4, P == 4, M % 4 == 0 — every HIPIE call site): one warp
//    owns (query, 4 heads); 8 lanes x float4 cover the 32 channels of a head, so every bilinear
//    tap is one fully used 128-byte line (64 B with a bf16 value map) and the per-(query, head)
//    locations / weights are loaded once, coalesced, and broadcast with shuffles instead of being
//    re-read by each channel lane.  All 64 taps of a head are independent loads in flight.
//  * optionally fused front half of MSDeformAttn.forward (softmax over L*P, reference-point +
//    offset arithmetic; .../ops/modules/ms_deform_attn.py:97-109) so the (N,Lq,M,L,P,2) location
//    tensor never exists in HBM, and the output can be emitted directly as the bf16 hi/lo split
//    consumed by the output_proj GEMM.
//  * generic path (any D/L/P, fp32 or fp64): one thread per output scalar; used by the
//    reference's own test shapes (ops/test.py: D=2, fp64).
#include "common.cuh"
#include "ptx.cuh"

namespace hipie {

// ------------------------------------------------------------------------------------------
// generic path
// ------------------------------------------------------------------------------------------
template <typename T>
__global__ void msda_generic_kernel(const T* __restrict__ value, const int64_t* __restrict__ shapes,
                                    const int64_t* __restrict__ lstart, const T* __restrict__ loc,
                                    const T* __restrict__ attw, T* __restrict__ out, int N, int S,
                                    int M, int D, int L, int Lq, int P) {
    const int64_t total = (int64_t)N * Lq * M * D;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (int64_t)gridDim.x * blockDim.x) {
        const int d = (int)(idx % D);
        const int m = (int)((idx / D) % M);
        const int64_t bq = idx / ((int64_t)D * M);  // b * Lq + q
        const int b = (int)(bq / Lq);
        const T* lp = loc + (bq * M + m) * (int64_t)L * P * 2;
        const T* wp = attw + (bq * M + m) * (int64_t)L * P;
        T acc = 0;
        for (int l = 0; l < L; ++l) {
            const int H = (int)shapes[2 * l], W = (int)shapes[2 * l + 1];
            const T* vbase = value + ((int64_t)b * S + lstart[l]) * M * D + (int64_t)m * D + d;
            const int64_t pix = (int64_t)M * D;
            for (int p = 0; p < P; ++p) {
                const T x = lp[(l * P + p) * 2] * W - (T)0.5;
                const T y = lp[(l * P + p) * 2 + 1] * H - (T)0.5;
                const T w = wp[l * P + p];
                if (y > -1 && x > -1 && y < H && x < W) {
                    const int y0 = (int)floor(y), x0 = (int)floor(x);
                    const T ly = y - y0, lx = x - x0, hy = 1 - ly, hx = 1 - lx;
                    T v1 = 0, v2 = 0, v3 = 0, v4 = 0;
                    if (y0 >= 0 && x0 >= 0) v1 = vbase[((int64_t)y0 * W + x0) * pix];
                    if (y0 >= 0 && x0 + 1 <= W - 1) v2 = vbase[((int64_t)y0 * W + x0 + 1) * pix];
                    if (y0 + 1 <= H - 1 && x0 >= 0) v3 = vbase[((int64_t)(y0 + 1) * W + x0) * pix];
                    if (y0 + 1 <= H - 1 && x0 + 1 <= W - 1)
                        v4 = vbase[((int64_t)(y0 + 1) * W + x0 + 1) * pix];
                    const T val = hy * hx * v1 + hy * lx * v2 + ly * hx * v3 + ly * lx * v4;
                    acc += w * val;
                }
            }
        }
        out[idx] = acc;
    }
}

// ------------------------------------------------------------------------------------------
// fast path
// ------------------------------------------------------------------------------------------
// value-map storage: 0 = fp32 (128-byte lines per tap and head), 1 = bf16, 2 = IEEE fp16 (64-byte lines: half the L2 -> L1 fill traffic
// that bounds the encoder calls; the precision map of DESIGN.md 3 adopts fp16 for the encoders' value maps)
template <int BF16V>
struct ValLoad;
template <>
struct ValLoad<0> {
    static __device__ __forceinline__ float4 ld(const void* base, int64_t elem_off) {
        return ldg_nc_f4(reinterpret_cast<const float*>(base) + elem_off);
    }
};
template <>
struct ValLoad<2> {
    static __device__ __forceinline__ float4 ld(const void* base, int64_t elem_off) {
        uint2 r;
        const __half* p = reinterpret_cast<const __half*>(base) + elem_off;
        asm volatile("ld.global.nc.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
        const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&r.x)), b = __half22float2(*reinterpret_cast<const __half2*>(&r.y));
        return make_float4(a.x, a.y, b.x, b.y);
    }
};
template <>
struct ValLoad<1> {
    static __device__ __forceinline__ float4 ld(const void* base, int64_t elem_off) {
        uint2 r;
        const __nv_bfloat16* p = reinterpret_cast<const __nv_bfloat16*>(base) + elem_off;
        asm volatile("ld.global.nc.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
        float4 o;
        o.x = __uint_as_float(r.x << 16);
        o.y = __uint_as_float(r.x & 0xffff0000u);
        o.z = __uint_as_float(r.y << 16);
        o.w = __uint_as_float(r.y & 0xffff0000u);
        return o;
    }
};

// FUSED: offs_logits rows are [M*L*P*2 offsets | M*L*P logits]; REFDIM in {2,4}.
// otherwise loc/attw are the reference operator's tensors.
template <int BF16V, bool FUSED, int REFDIM, bool SPLIT_OUT>
__global__ void __launch_bounds__(256)
msda_fast_kernel(const void* __restrict__ value, const int64_t* __restrict__ shapes,
                 const int64_t* __restrict__ lstart, const float* __restrict__ loc,
                 const float* __restrict__ attw, const float* __restrict__ refp,
                 float* __restrict__ out, __nv_bfloat16* __restrict__ out_hi,
                 __nv_bfloat16* __restrict__ out_lo, int N, int S, int M, int Lq) {
    constexpr int D = 32, L = 4, P = 4;
    const int lane = threadIdx.x & 31;
    const int hgroups = M >> 2;
    const int64_t warp_global = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwork = (int64_t)N * Lq * hgroups;
    if (warp_global >= nwork) return;
    // consecutive warps -> consecutive head groups of the same query, then next query
    const int hg = (int)(warp_global % hgroups);
    const int64_t bq = warp_global / hgroups;
    const int b = (int)(bq / Lq);
    const int hsub = lane >> 3, dsub = lane & 7;
    const int m = hg * 4 + hsub;

    int Hl[L], Wl[L];
    int64_t st[L];
#pragma unroll
    for (int l = 0; l < L; ++l) {
        Hl[l] = (int)__ldg(shapes + 2 * l);
        Wl[l] = (int)__ldg(shapes + 2 * l + 1);
        st[l] = __ldg(lstart + l);
    }

    // this lane owns points p0 = 2*dsub, p0+1 of head m (both on level dsub >> 1)
    float x0p, y0p, x1p, y1p, w0p, w1p;
    {
        const int lown = dsub >> 1;
        int Hown = Hl[0], Wown = Wl[0];
#pragma unroll
        for (int l = 1; l < L; ++l)
            if (lown == l) { Hown = Hl[l]; Wown = Wl[l]; }
        const float Wf = (float)Wown, Hf = (float)Hown;
        float4 o;
        float2 lg;
        if (FUSED) {
            const float* row = loc + bq * (int64_t)(M * L * P * 3);
            o = *reinterpret_cast<const float4*>(row + (hg * 4) * (L * P * 2) + lane * 4);
            lg = *reinterpret_cast<const float2*>(row + M * L * P * 2 + (hg * 4) * (L * P) + lane * 2);
            // softmax over the 16 logits of this head (8 lanes x 2)
            float mx = fmaxf(lg.x, lg.y);
#pragma unroll
            for (int s = 1; s < 8; s <<= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, s));
            float e0 = expf(lg.x - mx), e1 = expf(lg.y - mx);
            float sum = e0 + e1;
#pragma unroll
            for (int s = 1; s < 8; s <<= 1) sum += __shfl_xor_sync(0xffffffffu, sum, s);
            const float inv = 1.0f / sum;
            w0p = e0 * inv;
            w1p = e1 * inv;
            const float* rp = refp + (bq * L + lown) * REFDIM;
            float lx0, ly0, lx1, ly1;
            if (REFDIM == 2) {
                const float rx = rp[0], ry = rp[1];
                lx0 = rx + o.x / Wf; ly0 = ry + o.y / Hf;
                lx1 = rx + o.z / Wf; ly1 = ry + o.w / Hf;
            } else {
                const float rx = rp[0], ry = rp[1], rw = rp[2], rh = rp[3];
                lx0 = rx + o.x / (float)P * rw * 0.5f; ly0 = ry + o.y / (float)P * rh * 0.5f;
                lx1 = rx + o.z / (float)P * rw * 0.5f; ly1 = ry + o.w / (float)P * rh * 0.5f;
            }
            x0p = lx0 * Wf - 0.5f; y0p = ly0 * Hf - 0.5f;
            x1p = lx1 * Wf - 0.5f; y1p = ly1 * Hf - 0.5f;
        } else {
            const float* lrow = loc + (bq * M + hg * 4) * (int64_t)(L * P * 2);
            const float* wrow = attw + (bq * M + hg * 4) * (int64_t)(L * P);
            o = *reinterpret_cast<const float4*>(lrow + lane * 4);
            lg = *reinterpret_cast<const float2*>(wrow + lane * 2);
            w0p = lg.x; w1p = lg.y;
            x0p = o.x * Wf - 0.5f; y0p = o.y * Hf - 0.5f;
            x1p = o.z * Wf - 0.5f; y1p = o.w * Hf - 0.5f;
        }
    }

    // ---- tap preparation: this lane turns its two points into 4 element offsets + 4 fused weights each (attention
    //      weight x bilinear weight; out-of-range taps get weight 0 and a clamped in-range address, so the gather loop is
    //      branch free), staged in shared memory for the 8 lanes of the head group.
    extern __shared__ __align__(16) uint8_t msda_smem[];
    const int warp_in_blk = threadIdx.x >> 5;
    // per warp: 4 head groups x (16 points x 8 words + 4 pad words)  -> distinct banks for the 4 broadcast addresses
    constexpr int GROUP_WORDS = 16 * 8 + 4;
    uint32_t* wsm = reinterpret_cast<uint32_t*>(msda_smem) + warp_in_blk * 4 * GROUP_WORDS;
    const int pixstride_i = M * D;
    {
        const int lown = dsub >> 1;
        int Hown = Hl[0], Wown = Wl[0];
        int64_t stown = st[0];
#pragma unroll
        for (int l = 1; l < L; ++l)
            if (lown == l) { Hown = Hl[l]; Wown = Wl[l]; stown = st[l]; }
#pragma unroll
        for (int pp = 0; pp < 2; ++pp) {
            const float x = pp ? x1p : x0p, y = pp ? y1p : y0p, w = pp ? w1p : w0p;
            const float yf = floorf(y), xf = floorf(x);
            const float ly = y - yf, lx = x - xf, hy = 1.f - ly, hx = 1.f - lx;
            // clamp the integer corner so that int conversion is safe for wild offsets
            const int yi = (int)fminf(fmaxf(yf, -2.f), (float)Hown), xi = (int)fminf(fmaxf(xf, -2.f), (float)Wown);
            const bool inside = y > -1.f && x > -1.f && y < (float)Hown && x < (float)Wown;
            const bool t = inside && yi >= 0, btm = inside && yi + 1 <= Hown - 1, lft = xi >= 0, rgt = xi + 1 <= Wown - 1;
            const int yc0 = min(max(yi, 0), Hown - 1), yc1 = min(max(yi + 1, 0), Hown - 1);
            const int xc0 = min(max(xi, 0), Wown - 1), xc1 = min(max(xi + 1, 0), Wown - 1);
            const int base = (int)stown * pixstride_i + m * D;
            uint4 offs;
            offs.x = base + (yc0 * Wown + xc0) * pixstride_i;
            offs.y = base + (yc0 * Wown + xc1) * pixstride_i;
            offs.z = base + (yc1 * Wown + xc0) * pixstride_i;
            offs.w = base + (yc1 * Wown + xc1) * pixstride_i;
            float4 wt;
            wt.x = (t && lft) ? w * hy * hx : 0.f;
            wt.y = (t && rgt) ? w * hy * lx : 0.f;
            wt.z = (btm && lft) ? w * ly * hx : 0.f;
            wt.w = (btm && rgt) ? w * ly * lx : 0.f;
            uint32_t* dst = wsm + hsub * GROUP_WORDS + (dsub * 2 + pp) * 8;
            *reinterpret_cast<uint4*>(dst) = offs;
            *reinterpret_cast<float4*>(dst + 4) = wt;
        }
    }
    __syncwarp();

    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    const int64_t vb = (int64_t)b * S * pixstride_i + dsub * 4;
    const uint32_t* gsm = wsm + hsub * GROUP_WORDS;
#pragma unroll
    for (int p = 0; p < L * P; ++p) {
        const uint4 offs = *reinterpret_cast<const uint4*>(gsm + p * 8);
        const float4 wt = *reinterpret_cast<const float4*>(gsm + p * 8 + 4);
        const float4 v1 = ValLoad<BF16V>::ld(value, vb + offs.x);
        const float4 v2 = ValLoad<BF16V>::ld(value, vb + offs.y);
        const float4 v3 = ValLoad<BF16V>::ld(value, vb + offs.z);
        const float4 v4 = ValLoad<BF16V>::ld(value, vb + offs.w);
        acc.x += wt.x * v1.x + wt.y * v2.x + wt.z * v3.x + wt.w * v4.x;
        acc.y += wt.x * v1.y + wt.y * v2.y + wt.z * v3.y + wt.w * v4.y;
        acc.z += wt.x * v1.z + wt.y * v2.z + wt.z * v3.z + wt.w * v4.z;
        acc.w += wt.x * v1.w + wt.y * v2.w + wt.z * v3.w + wt.w * v4.w;
    }

    const int64_t o = bq * (int64_t)(M * D) + m * D + dsub * 4;
    if (SPLIT_OUT) {
        uint2 hi, lo;
        split2(acc.x, acc.y, hi.x, lo.x);
        split2(acc.z, acc.w, hi.y, lo.y);
        *reinterpret_cast<uint2*>(out_hi + o) = hi;
        if (out_lo) *reinterpret_cast<uint2*>(out_lo + o) = lo;
        if (out) *reinterpret_cast<float4*>(out + o) = acc;
    } else {
        *reinterpret_cast<float4*>(out + o) = acc;
    }
}

// ------------------------------------------------------------------------------------------
// encoder path (Lq == S, 2-d reference points, fused front half): value-map windows in shared memory
// ------------------------------------------------------------------------------------------
// The flat kernel above gathers every bilinear tap as a 128-byte line through L1: 89 M lines per encoder call at B = 8, two thirds
// of them missing L1 (ncu, round 1: L1 hit 36 %, L2 -> L1 fills at the L2 throughput cap).  In the encoder the queries ARE the
// pixels of the four levels and the learned offsets are a few pixels, so all taps of the queries inside one image region fall
// into a small window of every level.  One work item = (image, head, region): the region's windows of the four levels
// (region + halo, 32 channels of the head: 128 bytes per pixel) are brought into shared memory by four TMA box loads -- the
// hardware zero-fills what lies outside the level, which IS the zero padding of the bilinear sampling -- and the region's
// queries of all four levels gather from shared memory at one 128-byte wavefront per corner, conflict-free.  Taps that leave
// the window (large offsets) take the global path of the flat kernel, so the result does not depend on the halo.
// Same arithmetic, same summation order as msda_fast_kernel: results are bit-identical.
int make_tmap_f32_5d(CUtensorMap* out, const void* ptr, const uint64_t dims[5], const uint64_t strides_bytes[4], const uint32_t box[5]);

struct MsdaWinParams {
    const float* value;
    const float* offs_logits;     // (N, Lq, M*16*3)
    const float* refp;            // (N, Lq, 4, 2)
    float* out;
    __nv_bfloat16* out_hi;
    __nv_bfloat16* out_lo;
    int N, S, M;
    int H[4], W[4], lsi[4];
    int nty, ntx;                 // regions per image
    int ww[4], wh[4];             // window (TMA box) size per level, pixels
    int wbase[4];                 // byte offset of the level's window in shared memory
    int halo;
    int win_bytes;                // total bytes of the four windows (mbarrier transaction count)
};
struct MsdaWinMaps { CUtensorMap l[4]; };

constexpr int MW_THREADS = 512;                  // 16 warps: 64 (query, head) pairs in flight per step
constexpr int MW_GROUP_WORDS = 16 * 8 + 4;       // per (warp, quarter): 16 points x (4 offsets + 4 weights), padded
constexpr uint32_t MW_GLOBAL = 0x80000000u;      // record flag: offsets are global element offsets, not window byte offsets

template <bool SPLIT_OUT>
__global__ void __launch_bounds__(MW_THREADS, 1)
msda_win_kernel(const __grid_constant__ MsdaWinMaps maps, const MsdaWinParams p) {
    using namespace ptx;
    constexpr int D = 32, L = 4, P = 4;
    extern __shared__ uint8_t mw_raw[];
    // offset arithmetic (not an integer round trip) keeps the pointer in the shared address space: LDS / STS, not generic LD / ST
    uint8_t* smem = mw_raw + ((128u - (smem_u32(mw_raw) & 127u)) & 127u);
    uint32_t* recs = reinterpret_cast<uint32_t*>(smem + p.win_bytes);                      // [16 warps][4][MW_GROUP_WORDS]
    uint64_t* bar = reinterpret_cast<uint64_t*>(smem + p.win_bytes + (MW_THREADS / 32) * 4 * MW_GROUP_WORDS * 4);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, hsub = lane >> 3, dsub = lane & 7;
    const uint32_t win_s = smem_u32(smem);
    if (tid == 0) {
        for (int l = 0; l < L; ++l) prefetch_tmap(&maps.l[l]);
        mbar_init(bar, 1);
        fence_barrier_init();
    }
    __syncthreads();
    const int ntiles = p.nty * p.ntx;
    const int items = p.N * p.M * ntiles;
    const int pixstride = p.M * D;
    uint32_t phase = 0;
    for (int it = blockIdx.x; it < items; it += gridDim.x) {
        const int tile = it % ntiles, m = (it / ntiles) % p.M, b = it / (ntiles * p.M);
        const int ty = tile / p.ntx, tx = tile - ty * p.ntx;
        // region geometry: query rows / columns of every level inside the region, and the window origin of every level
        int ys[L], xs[L], th[L], tw[L], wx0[L], wy0[L], cum[L + 1];
        cum[0] = 0;
#pragma unroll
        for (int l = 0; l < L; ++l) {
            ys[l] = (ty * p.H[l] + p.nty - 1) / p.nty;
            xs[l] = (tx * p.W[l] + p.ntx - 1) / p.ntx;
            th[l] = ((ty + 1) * p.H[l] + p.nty - 1) / p.nty - ys[l];
            tw[l] = ((tx + 1) * p.W[l] + p.ntx - 1) / p.ntx - xs[l];
            cum[l + 1] = cum[l] + th[l] * tw[l];
            wx0[l] = (int)floorf((float)(tx * p.W[l]) / (float)p.ntx - 0.5f) - p.halo;
            wy0[l] = (int)floorf((float)(ty * p.H[l]) / (float)p.nty - 0.5f) - p.halo;
        }
        const int nq = cum[L];
        __syncthreads();                       // every warp is done with the previous item's windows
        if (tid == 0) {
            mbar_arrive_expect_tx(bar, (uint32_t)p.win_bytes);
#pragma unroll
            for (int l = 0; l < L; ++l) tma_load_5d(smem + p.wbase[l], &maps.l[l], bar, 0, m, wx0[l], wy0[l], b);
        }
        bool landed = false;
        // the front-half inputs of a group (offsets, logits, reference point: global loads with ~1 us latency) are fetched one
        // group ahead, so the latency hides behind the previous group's gather
        struct Fetch { float4 o; float2 lg; float rx, ry; int q; bool valid; };
        const int lown = dsub >> 1;
        auto fetch = [&](int g0) {
            Fetch f;
            const int qi = g0 + warp * 4 + hsub;
            f.valid = qi < nq;
            const int qc = f.valid ? qi : 0;
            int lq = 0;
#pragma unroll
            for (int l = 1; l < L; ++l) lq += (qc >= cum[l]) ? 1 : 0;
            int r = qc, twl = tw[0], ysl = ys[0], xsl = xs[0], Wl = p.W[0], base = p.lsi[0];
#pragma unroll
            for (int l = 1; l < L; ++l)
                if (lq == l) { r = qc - cum[l]; twl = tw[l]; ysl = ys[l]; xsl = xs[l]; Wl = p.W[l]; base = p.lsi[l]; }
            twl = max(twl, 1);
            f.q = base + (ysl + r / twl) * Wl + xsl + r % twl;      // query index inside the image (level-major, row-major)
            const int64_t bq = (int64_t)b * p.S + f.q;
            const float* row = p.offs_logits + bq * (int64_t)(p.M * L * P * 3);
            f.o = *reinterpret_cast<const float4*>(row + m * (L * P * 2) + dsub * 4);
            f.lg = *reinterpret_cast<const float2*>(row + p.M * L * P * 2 + m * (L * P) + dsub * 2);
            const float* rp = p.refp + (bq * L + lown) * 2;
            f.rx = rp[0];
            f.ry = rp[1];
            return f;
        };
        Fetch nxt = fetch(0);
        for (int g0 = 0; g0 < nq; g0 += MW_THREADS / 8) {
            const Fetch cur = nxt;
            if (g0 + MW_THREADS / 8 < nq) nxt = fetch(g0 + MW_THREADS / 8);
            const bool qvalid = cur.valid;
            const int64_t bq = (int64_t)b * p.S + cur.q;
            // ---- front half for head m: this lane owns points 2*dsub, 2*dsub+1 (level dsub >> 1) of its quarter's query
            int Hown = p.H[0], Wown = p.W[0], stown = p.lsi[0], wwown = p.ww[0], whown = p.wh[0], wbown = p.wbase[0], wx = wx0[0], wy = wy0[0];
#pragma unroll
            for (int l = 1; l < L; ++l)
                if (lown == l) { Hown = p.H[l]; Wown = p.W[l]; stown = p.lsi[l]; wwown = p.ww[l]; whown = p.wh[l]; wbown = p.wbase[l]; wx = wx0[l]; wy = wy0[l]; }
            const float Wf = (float)Wown, Hf = (float)Hown;
            const float4 o = cur.o;
            const float2 lg = cur.lg;
            float mx = fmaxf(lg.x, lg.y);
#pragma unroll
            for (int s = 1; s < 8; s <<= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, s));
            const float e0 = expf(lg.x - mx), e1 = expf(lg.y - mx);
            float sum = e0 + e1;
#pragma unroll
            for (int s = 1; s < 8; s <<= 1) sum += __shfl_xor_sync(0xffffffffu, sum, s);
            const float inv = 1.0f / sum;
            const float w0p = e0 * inv, w1p = e1 * inv;
            const float rx = cur.rx, ry = cur.ry;
            const float x0p = (rx + o.x / Wf) * Wf - 0.5f, y0p = (ry + o.y / Hf) * Hf - 0.5f;
            const float x1p = (rx + o.z / Wf) * Wf - 0.5f, y1p = (ry + o.w / Hf) * Hf - 0.5f;
            uint32_t* wsm = recs + (warp * 4 + hsub) * MW_GROUP_WORDS;
#pragma unroll
            for (int pp = 0; pp < 2; ++pp) {
                const float x = pp ? x1p : x0p, y = pp ? y1p : y0p, w = pp ? w1p : w0p;
                const float yf = floorf(y), xf = floorf(x);
                const float ly = y - yf, lx = x - xf, hy = 1.f - ly, hx = 1.f - lx;
                const int yi = (int)fminf(fmaxf(yf, -2.f), (float)Hown), xi = (int)fminf(fmaxf(xf, -2.f), (float)Wown);
                const bool inside = y > -1.f && x > -1.f && y < (float)Hown && x < (float)Wown;
                const bool inwin = xi >= wx && xi + 1 < wx + wwown && yi >= wy && yi + 1 < wy + whown;
                uint4 offs;
                float4 wt;
                if (inside && inwin) {
                    // all four corners are inside the staged window; corners outside the level read the TMA zero fill
                    const uint32_t o00 = (uint32_t)wbown + (uint32_t)(((yi - wy) * wwown + (xi - wx)) * 128);
                    offs = make_uint4(o00, o00 + 128u, o00 + (uint32_t)wwown * 128u, o00 + (uint32_t)wwown * 128u + 128u);
                    const bool t = yi >= 0, btm = yi + 1 <= Hown - 1, lft = xi >= 0, rgt = xi + 1 <= Wown - 1;
                    wt.x = (t && lft) ? w * hy * hx : 0.f;
                    wt.y = (t && rgt) ? w * hy * lx : 0.f;
                    wt.z = (btm && lft) ? w * ly * hx : 0.f;
                    wt.w = (btm && rgt) ? w * ly * lx : 0.f;
                } else {
                    const bool t = inside && yi >= 0, btm = inside && yi + 1 <= Hown - 1, lft = xi >= 0, rgt = xi + 1 <= Wown - 1;
                    const int yc0 = min(max(yi, 0), Hown - 1), yc1 = min(max(yi + 1, 0), Hown - 1);
                    const int xc0 = min(max(xi, 0), Wown - 1), xc1 = min(max(xi + 1, 0), Wown - 1);
                    const int base = stown * pixstride + m * D;
                    offs.x = MW_GLOBAL | (uint32_t)(base + (yc0 * Wown + xc0) * pixstride);
                    offs.y = (uint32_t)(base + (yc0 * Wown + xc1) * pixstride);
                    offs.z = (uint32_t)(base + (yc1 * Wown + xc0) * pixstride);
                    offs.w = (uint32_t)(base + (yc1 * Wown + xc1) * pixstride);
                    wt.x = (t && lft) ? w * hy * hx : 0.f;
                    wt.y = (t && rgt) ? w * hy * lx : 0.f;
                    wt.z = (btm && lft) ? w * ly * hx : 0.f;
                    wt.w = (btm && rgt) ? w * ly * lx : 0.f;
                }
                uint32_t* dst = wsm + (dsub * 2 + pp) * 8;
                *reinterpret_cast<uint4*>(dst) = offs;
                *reinterpret_cast<float4*>(dst + 4) = wt;
            }
            __syncwarp();
            if (!landed) {                     // first group of the item: the windows have to be in shared memory from here on
                mbar_wait(bar, phase);
                landed = true;
            }
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            const float* vb = p.value + (int64_t)b * p.S * pixstride + dsub * 4;
            const uint32_t ws = win_s + dsub * 16;
#pragma unroll
            for (int pt = 0; pt < L * P; ++pt) {
                const uint4 offs = *reinterpret_cast<const uint4*>(wsm + pt * 8);
                const float4 wt = *reinterpret_cast<const float4*>(wsm + pt * 8 + 4);
                float4 v1, v2, v3, v4;
                if (offs.x & MW_GLOBAL) {
                    v1 = ldg_nc_f4(vb + (offs.x & ~MW_GLOBAL));
                    v2 = ldg_nc_f4(vb + offs.y);
                    v3 = ldg_nc_f4(vb + offs.z);
                    v4 = ldg_nc_f4(vb + offs.w);
                } else {
                    asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v1.x), "=f"(v1.y), "=f"(v1.z), "=f"(v1.w) : "r"(ws + offs.x));
                    asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v2.x), "=f"(v2.y), "=f"(v2.z), "=f"(v2.w) : "r"(ws + offs.y));
                    asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v3.x), "=f"(v3.y), "=f"(v3.z), "=f"(v3.w) : "r"(ws + offs.z));
                    asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v4.x), "=f"(v4.y), "=f"(v4.z), "=f"(v4.w) : "r"(ws + offs.w));
                }
                acc.x += wt.x * v1.x + wt.y * v2.x + wt.z * v3.x + wt.w * v4.x;
                acc.y += wt.x * v1.y + wt.y * v2.y + wt.z * v3.y + wt.w * v4.y;
                acc.z += wt.x * v1.z + wt.y * v2.z + wt.z * v3.z + wt.w * v4.z;
                acc.w += wt.x * v1.w + wt.y * v2.w + wt.z * v3.w + wt.w * v4.w;
            }
            if (qvalid) {
                const int64_t oo = bq * (int64_t)(p.M * D) + m * D + dsub * 4;
                if (SPLIT_OUT) {
                    uint2 hi, lo;
                    split2(acc.x, acc.y, hi.x, lo.x);
                    split2(acc.z, acc.w, hi.y, lo.y);
                    *reinterpret_cast<uint2*>(p.out_hi + oo) = hi;
                    if (p.out_lo) *reinterpret_cast<uint2*>(p.out_lo + oo) = lo;
                } else {
                    *reinterpret_cast<float4*>(p.out + oo) = acc;
                }
            }
            __syncwarp();                      // the records of this group are consumed before the next group overwrites them
        }
        if (!landed) mbar_wait(bar, phase);    // (a region without queries still has to retire its TMA transaction)
        phase ^= 1;
    }
}

template <int BF16V, bool FUSED, int REFDIM, bool SPLIT>
static int launch_fast(const void* value, const int64_t* shapes, const int64_t* lstart,
                       const float* loc, const float* attw, const float* refp, float* out,
                       void* out_hi, void* out_lo, int N, int S, int M, int Lq, cudaStream_t st) {
    const int64_t warps = (int64_t)N * Lq * (M / 4);
    const int64_t blocks = (warps + 7) / 8;
    if (blocks == 0) return HIPIE_OK;
    msda_fast_kernel<BF16V, FUSED, REFDIM, SPLIT><<<(unsigned)blocks, 256, 8 * 4 * (16 * 8 + 4) * 4, st>>>(
        value, shapes, lstart, loc, attw, refp, out, (__nv_bfloat16*)out_hi,
        (__nv_bfloat16*)out_lo, N, S, M, Lq);
    HIPIE_CHECK_LAUNCH();
    return HIPIE_OK;
}

}  // namespace hipie

using namespace hipie;

extern "C" int hipie_msda_forward(const void* value, const int64_t* spatial_shapes,
                                  const int64_t* level_start_index, const void* sampling_loc,
                                  const void* attn_weight, void* out, int N, int S, int M, int D,
                                  int L, int Lq, int P, int dtype, int value_dtype, void* stream) {
    if (N >= 0 && Lq >= 0 && (int64_t)N * Lq == 0) return HIPIE_OK;   // empty batch / no queries
    HIPIE_CHECK_ARG(value && spatial_shapes && level_start_index && sampling_loc && attn_weight && out,
                    "hipie_msda_forward: null pointer argument");
    HIPIE_CHECK_ARG(N >= 0 && S > 0 && M > 0 && D > 0 && L > 0 && Lq >= 0 && P > 0,
                    "hipie_msda_forward: bad sizes N=%d S=%d M=%d D=%d L=%d Lq=%d P=%d", N, S, M, D, L, Lq, P);
    HIPIE_CHECK_ARG(dtype == HIPIE_F32 || dtype == HIPIE_F64, "hipie_msda_forward: dtype must be f32/f64");
    HIPIE_CHECK_ARG(value_dtype == dtype || (value_dtype == HIPIE_BF16 && dtype == HIPIE_F32),
                    "hipie_msda_forward: value_dtype %d incompatible with dtype %d", value_dtype, dtype);
    cudaStream_t st = (cudaStream_t)stream;
    if ((int64_t)N * Lq == 0) return HIPIE_OK;
    const bool fast = dtype == HIPIE_F32 && D == 32 && L == 4 && P == 4 && (M % 4) == 0 &&
                      (((uintptr_t)value | (uintptr_t)sampling_loc | (uintptr_t)attn_weight | (uintptr_t)out) & 15) == 0;
    if (fast) {
        if (value_dtype == HIPIE_BF16)
            return launch_fast<1, false, 2, false>(value, spatial_shapes, level_start_index,
                                                      (const float*)sampling_loc, (const float*)attn_weight,
                                                      nullptr, (float*)out, nullptr, nullptr, N, S, M, Lq, st);
        return launch_fast<0, false, 2, false>(value, spatial_shapes, level_start_index,
                                                   (const float*)sampling_loc, (const float*)attn_weight,
                                                   nullptr, (float*)out, nullptr, nullptr, N, S, M, Lq, st);
    }
    HIPIE_CHECK_ARG(value_dtype == dtype, "hipie_msda_forward: bf16 value map needs the D=32,L=4,P=4 fast path");
    const int64_t total = (int64_t)N * Lq * M * D;
    const int threads = 256;
    int64_t blocks = (total + threads - 1) / threads;
    const int64_t cap = (int64_t)num_sms() * 32;
    if (blocks > cap) blocks = cap;
    if (dtype == HIPIE_F32)
        msda_generic_kernel<float><<<(unsigned)blocks, threads, 0, st>>>(
            (const float*)value, spatial_shapes, level_start_index, (const float*)sampling_loc,
            (const float*)attn_weight, (float*)out, N, S, M, D, L, Lq, P);
    else
        msda_generic_kernel<double><<<(unsigned)blocks, threads, 0, st>>>(
            (const double*)value, spatial_shapes, level_start_index, (const double*)sampling_loc,
            (const double*)attn_weight, (double*)out, N, S, M, D, L, Lq, P);
    HIPIE_CHECK_LAUNCH();
    return HIPIE_OK;
}

extern "C" int hipie_msda_fused_forward(const void* value, const int64_t* spatial_shapes,
                                        const int64_t* level_start_index, const float* offs_logits,
                                        const float* reference_points, int ref_dim, void* out, int N,
                                        int S, int M, int D, int L, int Lq, int P, int value_dtype,
                                        int out_split_bf16, void* out_lo, void* stream) {
    HIPIE_CHECK_ARG(value && spatial_shapes && level_start_index && offs_logits && reference_points && out,
                    "hipie_msda_fused_forward: null pointer argument");
    HIPIE_CHECK_ARG(D == 32 && L == 4 && P == 4 && M > 0 && (M % 4) == 0,
                    "hipie_msda_fused_forward: only D=32, L=4, P=4, M%%4==0 (got D=%d L=%d P=%d M=%d)", D, L, P, M);
    HIPIE_CHECK_ARG(ref_dim == 2 || ref_dim == 4, "hipie_msda_fused_forward: ref_dim must be 2 or 4");
    HIPIE_CHECK_ARG(value_dtype == HIPIE_F32 || value_dtype == HIPIE_BF16 || value_dtype == HIPIE_F16, "bad value_dtype");
    cudaStream_t st = (cudaStream_t)stream;
    if ((int64_t)N * Lq == 0) return HIPIE_OK;
    float* of = out_split_bf16 ? nullptr : (float*)out;
    void* ohi = out_split_bf16 ? out : nullptr;
#define HIPIE_MSDA_GO(BV, RD, SP)                                                                   \
    return launch_fast<BV, true, RD, SP>(value, spatial_shapes, level_start_index, offs_logits,    \
                                         nullptr, reference_points, of, ohi, out_lo, N, S, M, Lq, st)
    if (value_dtype == HIPIE_BF16) {
        if (ref_dim == 2) { if (out_split_bf16) HIPIE_MSDA_GO(1, 2, true); else HIPIE_MSDA_GO(1, 2, false); }
        else { if (out_split_bf16) HIPIE_MSDA_GO(1, 4, true); else HIPIE_MSDA_GO(1, 4, false); }
    } else if (value_dtype == HIPIE_F16) {
        if (ref_dim == 2) { if (out_split_bf16) HIPIE_MSDA_GO(2, 2, true); else HIPIE_MSDA_GO(2, 2, false); }
        else { if (out_split_bf16) HIPIE_MSDA_GO(2, 4, true); else HIPIE_MSDA_GO(2, 4, false); }
    } else {
        if (ref_dim == 2) { if (out_split_bf16) HIPIE_MSDA_GO(0, 2, true); else HIPIE_MSDA_GO(0, 2, false); }
        else { if (out_split_bf16) HIPIE_MSDA_GO(0, 4, true); else HIPIE_MSDA_GO(0, 4, false); }
    }
#undef HIPIE_MSDA_GO
}


// Encoder form of the fused op: the level geometry comes from the HOST (the caller knows it; it sizes the TMA windows), Lq == S,
// 2-d reference points, fp32 value map.  Falls back to hipie_msda_fused_forward semantics by returning HIPIE_EUNSUPPORTED when
// the shapes do not fit (the caller then uses the flat kernel).
extern "C" int hipie_msda_encoder_forward(const void* value, const int* shapes_hw_host, const float* offs_logits,
                                          const float* reference_points, void* out, int N, int S, int M, int D, int L, int P,
                                          int out_split_bf16, void* out_lo, int halo, void* stream) {
    HIPIE_CHECK_ARG(value && shapes_hw_host && offs_logits && reference_points && out, "hipie_msda_encoder_forward: null pointer argument");
    HIPIE_CHECK_ARG(D == 32 && L == 4 && P == 4 && M > 0, "hipie_msda_encoder_forward: only D=32, L=4, P=4 (got D=%d L=%d P=%d)", D, L, P);
    if ((int64_t)N * S == 0) return HIPIE_OK;
    MsdaWinParams p;
    p.value = (const float*)value; p.offs_logits = offs_logits; p.refp = reference_points;
    p.out = out_split_bf16 ? nullptr : (float*)out;
    p.out_hi = out_split_bf16 ? (__nv_bfloat16*)out : nullptr;
    p.out_lo = (__nv_bfloat16*)out_lo;
    p.N = N; p.S = S; p.M = M;
    int tot = 0;
    for (int l = 0; l < 4; ++l) {
        p.H[l] = shapes_hw_host[2 * l]; p.W[l] = shapes_hw_host[2 * l + 1];
        HIPIE_CHECK_ARG(p.H[l] > 0 && p.W[l] > 0, "hipie_msda_encoder_forward: bad level shape");
        p.lsi[l] = tot;
        tot += p.H[l] * p.W[l];
    }
    HIPIE_CHECK_ARG(tot == S, "hipie_msda_encoder_forward: level shapes sum to %d, S = %d", tot, S);
    HIPIE_CHECK_ARG((int64_t)S * M * D < (1ll << 30), "hipie_msda_encoder_forward: value map too large for 31-bit element offsets");
    p.nty = (p.H[0] + 15) / 16; p.ntx = (p.W[0] + 15) / 16;       // regions of 16 x 16 finest-level queries
    const int rec_bytes = (MW_THREADS / 32) * 4 * MW_GROUP_WORDS * 4;
    int h = halo > 0 ? halo : 4;
    for (; h >= 2; --h) {
        int bytes = 0;
        for (int l = 0; l < 4; ++l) {
            p.ww[l] = (p.W[l] + p.ntx - 1) / p.ntx + 2 * h + 2;
            p.wh[l] = (p.H[l] + p.nty - 1) / p.nty + 2 * h + 2;
            p.wbase[l] = bytes;
            bytes += p.ww[l] * p.wh[l] * 128;
        }
        p.win_bytes = bytes;
        if (bytes + rec_bytes + 256 <= 224 * 1024 && p.ww[0] <= 256 && p.wh[0] <= 256) break;
    }
    if (h < 2) { set_error("hipie_msda_encoder_forward: level windows do not fit in shared memory"); return HIPIE_EUNSUPPORTED; }
    p.halo = h;
    MsdaWinMaps maps;
    for (int l = 0; l < 4; ++l) {
        const uint64_t dims[5] = {32, (uint64_t)M, (uint64_t)p.W[l], (uint64_t)p.H[l], (uint64_t)N};
        const uint64_t strides[4] = {128, (uint64_t)M * 128, (uint64_t)p.W[l] * M * 128, (uint64_t)S * M * 128};
        const uint32_t box[5] = {32, 1, (uint32_t)p.ww[l], (uint32_t)p.wh[l], 1};
        int rc = make_tmap_f32_5d(&maps.l[l], (const float*)value + (int64_t)p.lsi[l] * M * 32, dims, strides, box);
        if (rc) return rc;
    }
    const int smem = p.win_bytes + rec_bytes + 256 + 128;
    const int items = N * M * p.nty * p.ntx;
    const int grid = items < num_sms() ? items : num_sms();
    cudaStream_t st = (cudaStream_t)stream;
    if (out_split_bf16) {
        HIPIE_ENSURE_SMEM(msda_win_kernel<true>, smem);
        msda_win_kernel<true><<<grid, MW_THREADS, smem, st>>>(maps, p);
    } else {
        HIPIE_ENSURE_SMEM(msda_win_kernel<false>, smem);
        msda_win_kernel<false><<<grid, MW_THREADS, smem, st>>>(maps, p);
    }
    HIPIE_CHECK_LAUNCH();
    return HIPIE_OK;
}
