/*
 * hipie_b200 — C-ABI of the H100-native (sm_90a) HIPIE inference hot path.
 *
 * Every entry point is `extern "C"`, takes plain device pointers + sizes + a
 * CUDA stream (passed as void*; NULL = legacy default stream), never
 * allocates, never synchronises, and returns 0 on success or a negative
 * HIPIE_E* code.  hipie_last_error() returns a static, human-readable string
 * for the calling thread's last failure.
 *
 * Reference interfaces replaced (paths relative to /root/reference,
 * H: = projects/HIPIE/hipie/):
 *   hipie_msda_forward      <- ms_deform_attn_forward, pybind module
 *                              `MultiScaleDeformableAttention`
 *                              (H:models/deformable_detr/ops/src/vision.cpp:13-16,
 *                               ms_deform_attn.h:21-40,
 *                               cuda/ms_deform_attn_cuda.cu:20-78); the twin copy under
 *                              H:models/maskdino/pixel_decoder/ops/src/ is the same function.
 *   hipie_gemm_*            <- torch.nn.functional.linear call sites of the ViT / DETR /
 *                              BERT blocks (H:backbone/vit.py:67-83,212-230; timm Mlp) and
 *                              einsum("bqc,bchw->bqhw") of
 *                              H:models/maskdino/transformer_decoder/maskdino_decoder.py:520-529
 *   hipie_attention_*       <- Attention.forward + add_decomposed_rel_pos
 *                              (H:backbone/vit.py:67-83, H:backbone/utils.py:96-125),
 *                              nn.MultiheadAttention of the decoders, BiMultiHeadAttention
 *                              (H:models/deformable_detr/fuse_helper.py:54-139)
 *   hipie_layernorm_* / hipie_groupnorm_* <- nn.LayerNorm / nn.GroupNorm call sites
 *   hipie_condinst_*        <- dynamic_mask_with_coords (H:models/ddetrs_dn.py:1411-1502)
 *
 * dtype codes: 0 = float32, 1 = float64 (msda generic path only), 2 = bfloat16.
 */
#ifndef HIPIE_B200_H_
#define HIPIE_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define HIPIE_OK 0
#define HIPIE_EINVAL (-1)   /* bad argument (shape, dtype, alignment, null pointer) */
#define HIPIE_ECUDA (-2)    /* a CUDA runtime / driver call failed */
#define HIPIE_EUNSUPPORTED (-3)

#define HIPIE_F32 0
#define HIPIE_F64 1
#define HIPIE_BF16 2
#define HIPIE_F16 3   /* IEEE fp16 value map of hipie_msda_fused_forward (DESIGN.md 3) */

/* epilogue activation codes for hipie_gemm */
#define HIPIE_ACT_NONE 0
#define HIPIE_ACT_RELU 1
#define HIPIE_ACT_GELU 2      /* exact erf GELU (timm Mlp / nn.GELU default) */
#define HIPIE_ACT_SIGMOID 3
#define HIPIE_ACT_QUICK_GELU 4 /* x * sigmoid(1.702 x): OpenAI CLIP (open_clip model.py, QuickGELU) */

const char* hipie_last_error(void);
int hipie_abi_version(void);
/* Number of kernel launches issued through this library by the calling process. */
int64_t hipie_launch_count(void);
/* Process-wide tuning switches (tests / A-B measurements), all default 1.  "gemm_tma_store": row-major outputs leave through TMA stores;
 * "gemm_fast_transposed": vectorised epilogue of the transposed fp16 plane (V^T); "ln_bulk": LayerNorm rows staged by bulk copies;
 * "ln_grid_cap": LayerNorm grid capped at the resident CTAs (rows grid-strided).  Unknown names return HIPIE_EINVAL. */
int hipie_set_option(const char* name, int value);

/* ------------------------------------------------------------------------------------------
 * Multi-scale deformable attention, forward.
 *   value             (N, S, M, D)        dtype, contiguous, device
 *   spatial_shapes    (L, 2) int64 (H_l, W_l), device
 *   level_start_index (L,)   int64, device
 *   sampling_loc      (N, Lq, M, L, P, 2) dtype, (x, y) normalised to [0,1], device
 *   attn_weight       (N, Lq, M, L, P)    dtype, device
 *   out               (N, Lq, M*D)        dtype, device; fully overwritten
 * dtype: HIPIE_F32 (fast path when D == 32, generic otherwise) or HIPIE_F64 (generic).
 * value_dtype: dtype of `value` storage; HIPIE_BF16 allowed only with dtype == HIPIE_F32
 *              (fast mode: bf16 value map, fp32 locations/weights/accumulation/output).
 * ------------------------------------------------------------------------------------------ */
int hipie_msda_forward(const void* value, const int64_t* spatial_shapes,
                       const int64_t* level_start_index, const void* sampling_loc,
                       const void* attn_weight, void* out, int N, int S, int M, int D, int L,
                       int Lq, int P, int dtype, int value_dtype, void* stream);

/* Fused front half of MSDeformAttn.forward (H:.../ops/modules/ms_deform_attn.py:97-109):
 * takes the raw `sampling_offsets` / `attention_weights` linear outputs packed as one
 * (N*Lq, M*L*P*3) fp32 matrix [offsets (M,L,P,2) | logits (M,L*P)], the reference points
 * (N, Lq, L, 2|4), does softmax over L*P, builds the sampling locations and runs the core op. */
int hipie_msda_fused_forward(const void* value, const int64_t* spatial_shapes,
                             const int64_t* level_start_index, const float* offs_logits,
                             const float* reference_points, int ref_dim, void* out, int N, int S,
                             int M, int D, int L, int Lq, int P, int value_dtype,
                             int out_split_bf16, void* out_lo, void* stream);

/* ------------------------------------------------------------------------------------------
 * wgmma GEMM:  C[M,N] = act( A[M,K] . W[N,K]^T + bias[N] ) * colscale[N] + residual[M,N]
 * A and W are bf16 "split" operands: a_hi/a_lo and w_hi/w_lo (lo may be NULL when prec == 1).
 *   prec == 1 : C = Ahi.Whi                      (plain bf16, fp32 accumulate)
 *   prec == 3 : C = Ahi.Whi + Ahi.Wlo + Alo.Whi  (bf16x3 split, ~fp32 accuracy)
 *   prec == 2 : C = A.W, both ONE IEEE fp16 plane  (contractions normalised by a softmax, DESIGN.md 3)
 *   prec == 4 : C = A.Whi + A.Wlo, A ONE fp16 plane, W fp16 hi + lo (a_lo NULL): the weight exact to ~2^-22, the activation
 *               rounded to fp16 once -- the qkv linears, whose outputs the fp16 attention rounds to fp16 anyway
 *   prec == 6 : C = Ah.Wh + 2^-14 (a8 . w8^T): the fp16 hi x hi product in one 16-bit pass, both cross terms Ah.Wl + Al.Wh in ONE
 *               e4m3 pass over 2K (kind::f8f6f4 runs at twice the 16-bit rate): two pass-equivalents for ~2^-15.5 relative error
 *               per product, the class of the three-pass bf16 split (DESIGN.md 3).  |A| must stay below 448 * 2 (e4m3 saturates),
 *               |W| below 28; hipie_split_f16_e4m3 builds the planes.
 * Row strides (in elements) lda / ldw / ldc allow strided sub-matrices; K % 8 == 0,
 * all base pointers 16-byte aligned.  Outputs (any subset, NULL to skip):
 *   c_f32 (fp32), c_hi / c_lo (bf16 split of the fp32 result, for feeding the next GEMM),
 *   c_bits: 1 bit per element (result > threshold), row-major, N padded to 32 — used by the
 *           mask-embed contraction fused with sigmoid+threshold.
 * batch: number of independent problems; *_bstride are element strides between them.
 * ------------------------------------------------------------------------------------------ */
typedef struct hipie_gemm_args {
    const void* a_hi; const void* a_lo; int64_t lda; int64_t a_bstride;
    const void* w_hi; const void* w_lo; int64_t ldw; int64_t w_bstride;
    const float* bias;        /* [N] or NULL */
    const float* colscale;    /* [N] or NULL (layer-scale gamma) */
    const float* residual;    /* [M, ldr] fp32 or NULL */
    int64_t ldr; int64_t r_bstride;
    float* c_f32; void* c_hi; void* c_lo; int64_t ldc; int64_t c_bstride;
    uint32_t* c_bits; float bits_threshold;
    int M, N, K, batch;
    int act;                  /* HIPIE_ACT_* */
    int prec;                 /* 3: bf16 hi/lo planes, Ah.Wh + Ah.Wl + Al.Wh (fp32-class); 1: bf16 hi planes, one pass;
                                 2: a_hi / w_hi are IEEE fp16 planes, one pass (the parity-grade single-pass mode, DESIGN.md 3);
                                 4: a_hi one fp16 plane, w_hi / w_lo fp16 hi + lo planes, two passes */
    float alpha;              /* scales the accumulator before bias (1.0f default) */
    int transposed;           /* 1: C (and residual, c_hi/lo) addressed as [col * ld + row]; c_bits is then packed along M:
                                 bits[b][col][row/32].  0: c_bits (needs N % 16 == 0) is packed along N: bits[b][row][col/32] */
    const int32_t* c_row_map; /* optional (non-transposed only): GEMM row r is stored to / takes its residual
                                 from row c_row_map[r]; negative entries are skipped (window un-partition) */
    int t_row_group;          /* transposed only, 0 = off: GEMM row r is stored at position r + (r / t_row_group) * t_row_pad of */
    int t_row_pad;            /* each output column (groups of rows padded apart, e.g. 196-token windows at a 200 pitch)     */
    int relu_after_residual;  /* 1: ReLU applied AFTER the residual add (ResNet bottleneck: relu(conv3(x) + shortcut)); `act` is applied before */
    int c_fp16;               /* 1: c_hi receives IEEE fp16 values (one plane, c_lo must be NULL): operands of the single-pass fp16
                                 contractions (attention QK^T / PV, DESIGN.md 3); 0: bf16 hi (+ lo) planes */
    /* prec 6 (fp16 + e4m3 split, see below): e4m3 planes of the operands, row strides in bytes */
    /* The e4m3 planes hold two "slots" per element, interleaved in 32-column groups: byte (k / 32) * 64 + k % 32 = slot 0 of column k,
       +32 = slot 1 (a producer's 32-column chunk is one 64-byte segment); K % 32 == 0. */
    const void* a8; int64_t lda8;   /* (M, 2K): slot 0 = e4m3(Ah), slot 1 = e4m3(2^10 (A - Ah)), Ah = fp16(A) = a_hi */
    const void* w8; int64_t ldw8;   /* (N, 2K): slot 0 = e4m3(2^14 (W - Wh)), slot 1 = e4m3(2^4 Wh), Wh = fp16(W) = w_hi */
    void* c8; int64_t ldc8;         /* optional with c_fp16: the result's own e4m3 planes (M, 2N) in the a8 layout, so that the
                                       output feeds the next prec-6 GEMM (fc1 -> fc2); needs N % 32 == 0 */
} hipie_gemm_args;

/* Encoder form of the fused MSDeformAttn op (Lq == S: the queries are the pixels of the four levels; 2-d reference points; fp32
 * value map): one work item = (image, head, 16x16-pixel region of the finest level); the region's windows of all four levels are
 * staged in shared memory by TMA (zero fill outside a level = the sampling's zero padding) and the region's queries gather from
 * shared memory; taps outside the halo take the global path, so results equal hipie_msda_fused_forward bit for bit.
 *   shapes_hw_host: HOST array of 4 (H_l, W_l) pairs (sizes the TMA boxes); halo: pixels around the region (0 = default 4, reduced
 *   automatically until the windows fit).  Returns HIPIE_EUNSUPPORTED when the windows cannot fit: use the flat kernel then. */
int hipie_msda_encoder_forward(const void* value, const int* shapes_hw_host, const float* offs_logits, const float* reference_points,
                               void* out, int N, int S, int M, int D, int L, int P, int out_split_bf16, void* out_lo, int halo,
                               void* stream);

int hipie_gemm(const hipie_gemm_args* args, void* stream);

/* fp32 -> bf16 hi (+ lo = bf16(x - hi)) split of a contiguous array of n elements. */
int hipie_split_bf16(const float* x, void* hi, void* lo, int64_t n, void* stream);

/* fp32 (rows, cols) -> the operand planes of a prec-6 hipie_gemm: h16 (rows, cols) fp16 and p8 (rows, 2 * cols) e4m3.
 * weight == 0 (activation A): slots e4m3(h), e4m3(2^10 (x - h));  weight == 1 (W): slots e4m3(2^14 (x - h)), e4m3(2^4 h); the slots are
 * interleaved in 32-column groups (see hipie_gemm_args.a8); cols % 32 == 0. */
int hipie_split_f16_e4m3(const float* x, void* h16, void* p8, int64_t rows, int cols, int weight, void* stream);

/* LayerNorm over the last dim C of x[rows, C] (fp32 in).  Outputs: y_f32 and/or bf16 split
 * (y_hi, y_lo).  Optional `add` tensor is added to x before normalisation and the sum is
 * written to sum_out (residual stream), matching post-LN layers: y = LN(x + add). */
int hipie_layernorm(const float* x, const float* add, const float* gamma, const float* beta,
                    float eps, float* sum_out, float* y_f32, void* y_hi, void* y_lo,
                    int64_t rows, int C, const int32_t* out_row_map, void* stream);
/* Same LayerNorm with the normalised rows written as ONE IEEE fp16 plane: the A operand of a prec-4 (two-pass fp16) hipie_gemm
 * -- the qkv linears of the ViT blocks (H:backbone/vit.py:67-70), whose outputs are rounded to fp16 for the attention anyway.
 * y_e4m3 (optional, rows x 2C): additionally the e4m3 planes [e4m3(h) | e4m3(2^10 (y - h))] of a prec-6 GEMM's A operand (norm2 -> fc1). */
int hipie_layernorm_f16(const float* x, const float* add, const float* gamma, const float* beta,
                        float eps, float* sum_out, float* y_f32, void* y_f16, void* y_e4m3,
                        int64_t rows, int C, const int32_t* out_row_map, void* stream);

/* GroupNorm(G) over NHWC fp32 (N, HW, C) with per-sample strides, optional fused ReLU and a
 * tensor added after the normalisation; stats_ws: 2*N*G doubles of scratch. */
int hipie_groupnorm_nhwc(const float* x, const float* gamma, const float* beta, float eps,
                         const float* post_add, float* y_f32, void* y_hi, void* y_lo, double* stats_ws,
                         int N, int HW, int C, int G, int relu, int64_t x_bstride, int64_t y_bstride,
                         int64_t add_bstride, void* stream);

/* out = a + b (b may be NULL) as fp32 and/or bf16 split. */
int hipie_add_split(const float* a, const float* b, float* sum_f32, void* hi, void* lo, int64_t n,
                    void* stream);
/* PatchEmbed im2col fused with (x - mean) / std: img (B,3,H,W) -> rows (B*(H/P)*(W/P), 3*P*P). */
int hipie_patchify(const float* img, void* hi, void* lo, int B, int H, int W, int P,
                   const float* mean3_host, const float* std3_host, void* stream);
/* NHWC im2col for k x k convolutions: rows (B*Ho*Wo, k*k*C), column order (ky, kx, c). */
int hipie_im2col_nhwc(const float* x, void* hi, void* lo, int B, int H, int W, int C, int ksz,
                      int stride, int pad, void* stream);
/* ConvTranspose2d(k=2,s=2) pixel shuffle: (B*H*W, 4*C) [dy,dx,c] -> NHWC (B,2H,2W,C). */
int hipie_pixel_shuffle2(const float* g, float* y, void* hi, void* lo, int B, int H, int W, int C,
                         void* stream);
int hipie_maxpool2_nhwc(const float* x, float* y, void* hi, void* lo, int B, int H, int W, int C,
                        void* stream);
/* F.max_pool2d(kernel 3, stride 2, padding 1) on NHWC fp32 (ResNet stem); output (B, (H-1)/2+1, (W-1)/2+1, C) fp32 and/or bf16 split. */
int hipie_maxpool3x3s2_nhwc(const float* x, float* y, void* hi, void* lo, int B, int H, int W, int C, void* stream);
/* p = softmax(clamp(x [- rowmax], +-clampv) + colbias[row / rows_per_batch, :]) over the last dim. */
/* out_fp16 = 1: the probabilities are written as ONE IEEE fp16 plane (hi; lo NULL) for the single-pass fp16 contractions. */
int hipie_row_softmax(const float* x, const float* colbias, int64_t rows, int64_t rows_per_batch,
                      int n, float clampv, int sub_rowmax, void* hi, void* lo, float* p_f32,
                      int out_fp16, void* stream);

/* ------------------------------------------------------------------------------------------
 * Fused multi-head attention with optional decomposed relative-position bias
 * (H:backbone/utils.py:96-125) and optional additive key mask.
 *   q, k, v : bf16 split planes (hi, lo), logical shape (B, T, H, hd) with element strides
 *             given explicitly so the packed qkv GEMM output can be consumed in place.
 *   rel_h   : (B, H, Tq, kh) fp32 or NULL ; rel_w : (B, H, Tq, kw) fp32 or NULL ; Tk = kh*kw
 *   key_bias: (B, Tk) fp32 additive (0 / -inf style) or NULL ; key_mask: per-(batch, query) bit mask over the keys or NULL
 *   out     : (B, Tq, H*hd) fp32 and/or bf16 split.
 * scale is applied to q.k^T before the bias (reference: (q*scale) @ k^T + rel).
 * ------------------------------------------------------------------------------------------ */
typedef struct hipie_attn_args {
    const void* q_hi; const void* q_lo; const void* k_hi; const void* k_lo;
    const void* v_hi; const void* v_lo;
    int64_t q_bs, q_ts, q_hs;   /* element strides: batch, token, head (q) */
    int64_t k_bs, k_ts, k_hs;
    int64_t v_bs, v_ts, v_hs;
    const float* rel_h; const float* rel_w; int kh, kw;
    const float* key_bias;
    float* out_f32; void* out_hi; void* out_lo; int64_t o_bs, o_ts;
    int B, H, Tq, Tk, hd;
    float scale;
    int prec;
    const uint32_t* key_mask;   /* optional (B, Tq, ceil(Tk / 32)) bit words shared by all heads: bit k of a query's row set = key k is
                                 * masked OUT for that query (nn.MultiheadAttention's boolean attn_mask; MaskCLIP's per-query patch
                                 * masks open_vocab/clip.py:288-332, the causal mask of the CLIP text transformer) */
} hipie_attn_args;

int hipie_attention(const hipie_attn_args* args, void* stream);

/* wgmma flash attention for the ViT-H blocks (Attention.forward + add_decomposed_rel_pos, backbone/vit.py:67-83,
 * backbone/utils.py:96-125), hd == 80.  Two modes, selected by the shapes:
 *   global : T % 256 == 0, optional decomposed rel-pos bias with kw == 64 (1024-pixel inputs) or kw == 80 (1280-pixel inputs; then
 *            also T % 320 == 0), kh * kw == T; one CTA per 128 queries.  Other grids: HIPIE_EINVAL (callers use hipie_attention).
 *   window : T == 196 with kh == kw == 14 (the 14 x 14 windows; B = number of windows): two CTAs of 128 query rows per
 *            (window, head), the 60 padding query rows skip their stores and the 60 padding keys of the last 64-key tile are masked.
 * q / k are bf16 planes viewed as (B, T, width) rows (token stride *_ts, batch stride *_bs, head h at columns
 * [*_col0 + 80 h, +80)); vt is V transposed, (H*80, B*T) planes with row stride vt_ld (the qkv GEMM emits it with transposed=1);
 * in window mode every window sits at a 200-column pitch, (H*80, B*200), with zero pad columns (t_row_group = 196,
 * t_row_pad = 4 of hipie_gemm).  rel_h (B, H, T, kh) and rel_w (B, H, T, kw) fp32.  Output (B, T, H*80) fp32 and/or bf16 split.
 * prec: 3 = bf16 hi/lo planes, three MMA passes; 1 = bf16 hi planes, one pass; 2 = ONE IEEE fp16 plane per operand (the `*_hi`
 * pointers; hipie_gemm with c_fp16 = 1 emits them) and fp16 probabilities, one pass -- the parity-grade single-pass mode. */
int hipie_attention_tc(const void* q_hi, const void* q_lo, int64_t q_bs, int64_t q_ts, int q_col0, int q_width,
                       const void* k_hi, const void* k_lo, int64_t k_bs, int64_t k_ts, int k_col0, int k_width,
                       const void* vt_hi, const void* vt_lo, int64_t vt_ld, const float* rel_h, const float* rel_w,
                       int kh, int kw, float* out_f32, void* out_hi, void* out_lo, int64_t o_bs, int64_t o_ts, int B,
                       int H, int T, int hd, float scale, int prec, void* stream);

/* Same attention, output written as the operand planes of a prec-6 hipie_gemm (the proj linear, H:backbone/vit.py:82): out_f16
 * (B, T, H*hd) ONE fp16 plane and out_e4m3 (B*T, 2*H*hd) = [e4m3(h) | e4m3(2^10 (o - h))]; contiguous outputs (o_ts == H*hd). */
int hipie_attention_tc_planes(const void* q_hi, const void* q_lo, int64_t q_bs, int64_t q_ts, int q_col0, int q_width,
                              const void* k_hi, const void* k_lo, int64_t k_bs, int64_t k_ts, int k_col0, int k_width,
                              const void* vt_hi, const void* vt_lo, int64_t vt_ld, const float* rel_h, const float* rel_w,
                              int kh, int kw, float* out_f32, void* out_f16, void* out_e4m3, int64_t o_bs, int64_t o_ts, int B,
                              int H, int T, int hd, float scale, int prec, void* stream);

/* rel[b,h,q,j] = sum_c q[b,q,h,c] * table[idx(q,j), c] for the decomposed rel-pos bias.
 * axis 0: height (idx from q // qw), axis 1: width (q % qw).  table: (2*max(q,k)-1, hd) fp32,
 * table_t: get_rel_pos output (H:backbone/utils.py:63-93) pre-transposed to (qsize, hd, ksize) fp32.
 * q is read as hi (+ lo) bf16 planes. */
int hipie_relpos_bias(const void* q_hi, const void* q_lo, int64_t q_bs, int64_t q_ts, int64_t q_hs,
                      const float* table_t, int axis, int qh, int qw, int ksize, float* rel,
                      int B, int H, int hd, void* stream);

/* Tensor-core variant: table as bf16 hi/lo planes of the (qsize, ksize, hd) get_rel_pos output (K-major, no
 * transpose); one CTA per (coordinate, head, batch) group, mma.sync bf16x3. */
int hipie_relpos_bias_tc(const void* q_hi, const void* q_lo, int64_t q_bs, int64_t q_ts, int64_t q_hs,
                         const void* table_hi, const void* table_lo, int axis, int qh, int qw, int ksize,
                         float* rel, int B, int H, int hd, void* stream);
/* Same with q as ONE fp16 plane and the table as fp16 hi/lo planes (q.Rh + q.Rl, mma.sync f16): the rel-pos companion of the
 * single-pass fp16 attention. */
int hipie_relpos_bias_tc_f16(const void* q_f16, int64_t q_bs, int64_t q_ts, int64_t q_hs, const void* table_hi, const void* table_lo,
                             int axis, int qh, int qw, int ksize, float* rel, int B, int H, int hd, void* stream);

/* CondInst dynamic mask head, fused (H:models/ddetrs_dn.py:1390-1502,1806-1870):
 *   feats  (B, Hf*Wf, 8) NHWC fp32, params (B, Q, 169) fp32, ref_px (B, Q, 2) fp32 (pixels)
 *   out    (B, Q, 2*Hf, 2*Wf) fp32 mask logits after aligned_bilinear(x2). */
int hipie_condinst_masks(const float* feats, const float* params, const float* ref_px, float* out,
                         int B, int Q, int Hf, int Wf, int stride, void* stream);

/* Fused semantic + panoptic post-processing for one image (replaces the upsample / sigmoid / einsum / argmax / area chain of
 * projects/HIPIE/hipie/models/hipie_img.py:880-1023: semantic_inference + the tensor part of panoptic_inference).
 *   masks  (Q, h, w) f32   mask logits at 1/stride resolution (stride must be 4)
 *   pt_hi, pt_lo (ceil8(C) [10 or 17 rows of 8], Qpad) bf16  class probabilities transposed, bf16 hi/lo split, zero padded
 *   scores (Qpad) f32      per-query max class probability, 0 for queries that are not kept (score <= threshold / padding)
 *   sem    (C, Hc, Wc) f32 out: sum_q prob[q,c] * sigmoid(up(masks[q]))      (crop of the 4x upsampled map)
 *   ids    (Hc, Wc) i32    out: -1 if no query is kept, else 2*q + (sigmoid_q >= 0.5), q = argmax_q score_q * sigmoid_q
 *   areas  (3, Q) i32      out: [pixels won by q, pixels with sigmoid_q >= 0.5, pixels won by q with sigmoid_q >= 0.5] */
int hipie_seg_postprocess(const float* masks, const void* pt_hi, const void* pt_lo, const float* scores, float* sem, int* ids,
                          int* areas, int Q, int Qpad, int C, int h, int w, int stride, int Hc, int Wc, void* stream);

/* Instance masks of the kept detections (hipie_img.py:1003-1007): out[n, y, x] = sigmoid(bilinear_x4(masks[n]))[y, x] > threshold
 * for the (Hc, Wc) crop; masks (N, h, w) f32 logits at 1/4 resolution, out (N, Hc, Wc) one byte per pixel (torch.bool layout). */
int hipie_upsample_threshold(const float* masks, void* out_u8, int N, int h, int w, int stride, int Hc, int Wc,
                             float threshold, void* stream);

/* Sine embedding of box reference points (deformable_transformer_dino.py:636-670 get_sine_pos_embed; maskdino/utils/utils.py:74-100):
 * pos (rows, 4) = (x, y, w, h) f32 with row stride ld -> (rows, 512) = [emb(y) | emb(x) | emb(w) | emb(h)], 128 features each,
 * temperature 1e4, scale 2*pi.  out f32 and/or bf16 hi/lo planes (operand of the ref_point_head MLP). */
int hipie_sine_embed(const float* pos, int64_t ld, int64_t rows, float* out, void* hi, void* lo, void* stream);

/* ---- device-side selection steps of the inference post-processing (projects/HIPIE/hipie/hipie_img.py:587-657, 1025-1052) ----
 * hipie_class_scores: token -> class pooling of grounding logits (`convert_grounding_to_od_logits`).
 *   logits (R, Lt) f32 | tok (C, maxlen) i32 token indices of each class, cnt (C) i32 tokens per class (0 = class not in the
 *   positive map: score 0) | masked (C) i8 or NULL: 1 = class forced to -9999 (mode FG: stuff classes, mode BG: thing classes)
 *   iou (R) f32 logits or NULL | max_pool: 0 mean, 1 max over the class's tokens
 *   scores (R, C) f32 out | prob (R, C) f32 out or NULL: sqrt(sigmoid(score) * sigmoid(iou)) (sigmoid(score) if iou NULL)
 *   row_max (R) f32 / row_arg (R) i32 out or NULL: max / first argmax of prob over the classes (the NMS keys). */
int hipie_class_scores(const float* logits, const int* tok, const int* cnt, const int8_t* masked, const float* iou,
                       float* scores, float* prob, float* row_max, int* row_arg, int R, int Lt, int C, int maxlen,
                       int max_pool, void* stream);

/* hipie_batched_nms: torchvision.ops.batched_nms semantics (coordinate-offset trick: box + cls * (max_coord + 1), greedy in
 * decreasing score, IoU = inter / (a + b - inter) > threshold), one launch for B images.
 *   boxes (B, N, 4) f32 (cx, cy, w, h) | scores (B, N) f32 | cls (B, N) i32
 *   keep (B, N) i32 out: kept indices in decreasing score order, -1 padded | nkeep (B) i32 out.  N <= 1216 (the pair bit matrix lives in shared memory). */
int hipie_batched_nms(const float* boxes_cxcywh, const float* scores, const int* cls, int* keep, int* nkeep, int B, int N,
                      float iou_threshold, void* stream);

/* hipie_nms_sorted: greedy single-class NMS (torchvision.ops.nms: IoU = inter / (a + b - inter) > threshold, area = (x2 - x1) * (y2 - y1))
 * of N <= 32768 boxes already sorted by decreasing score (ties in the order the caller chose).
 *   boxes (N, 4) f32 xyxy, 16-byte aligned | mask_ws: device workspace of ws_words >= N * ceil(N / 64) u64 (the pair bit matrix)
 *   keep (N) i32 out: kept positions in the sorted order, ascending (the first nkeep are written) | nkeep (1) i32 out.  With N = 0
 *   only nkeep is needed (set to 0). */
int hipie_nms_sorted(const float* boxes_xyxy, int N, float iou_threshold, unsigned long long* mask_ws, int64_t ws_words, int* keep,
                     int* nkeep, void* stream);

/* hipie_topk: k largest of each row, values descending, lowest index first among equal values (torch.topk, largest=True).
 *   values: row r starts at values + r * row_stride; its length is n, or min(n, n_rows[r] * n_cols_per_row) when n_rows != NULL
 *   (a compacted (rows x cols) matrix whose valid row count lives on the device).  out_val (R, k) f32, out_idx (R, k) i32;
 *   rows shorter than k are padded with (-inf, -1).  k <= 1024. */
int hipie_topk(const float* values, int64_t row_stride, const int* n_rows, int n_cols_per_row, int R, int n, int k,
               float* out_val, int* out_idx, void* stream);

/* ---- MaskCLIP re-scoring (SURVEY a22 / f2: projects/HIPIE/hipie/open_vocab/clip.py:243-383, hipie_img.py:592-609,735-747,811-868) ----
 * The ViT-L/14 forward itself runs on hipie_gemm (QuickGELU epilogue) / hipie_layernorm / hipie_attention (key_mask); these cover
 * the steps around it.
 * hipie_maskclip_patch_mask: per-query patch masks of the mask tokens (clip.py:288-324).  masks (Q, h, w) f32 logits; up = 1: the
 *   maps are resized to S x S directly (hipie_img.py:599-602 passes the 1/4-resolution maps); up = 4: they are first upsampled x4 and
 *   cropped to (Hc, Wc) (hipie_img.py:733-741), evaluated on the fly.  For key = key_offset + patch: bit set in
 *   bits[q * row_words + key / 32] when max_pool_PxP(sigmoid(resized)) < 0.5, i.e. the patch is masked OUT; the rows are zeroed first.
 * hipie_clip_patches: image (3, H, W) f32 in 0..1 -> bilinear resize to S x S, (x - mean) / std, patch rows (S/P)^2 x (3 P P) in
 *   Conv2d weight order as bf16 hi/lo planes with row stride ld (the A operand of the patch-embedding GEMM).
 * hipie_clip_fuse: raw (R, Np) = mask_embed . unit(text_embed)^T; seg (C + 1) prompt offsets per class; scores (R, C) the model's
 *   class scores (-9999 = masked class), temp > 0: softmax(sigmoid(score) / temp), 0: sigmoid(score); overlap (C) i8 1 = class seen
 *   in training (weight alpha, else beta); agg_add 0 = geometric 'MUL', 1 = arithmetic 'ADD' (hipie_img.py:845-866).
 *   mode 0: out = fused log-probabilities; mode 1: out = sqrt(sigmoid(fused)^fg_a * sigmoid(iou)^fg_b) * [scores[0, c] != -9999]
 *   and its row max / first argmax; mode 2: out = softmax(fused) over the classes. */
int hipie_maskclip_patch_mask(const float* masks, int Q, int h, int w, int up, int Hc, int Wc, int S, int P, uint32_t* bits,
                              int row_words, int key_offset, void* stream);
int hipie_clip_patches(const float* image, int H, int W, int S, int P, const float* mean3, const float* std3, void* hi, void* lo,
                       int ld, void* stream);
int hipie_clip_fuse(const float* raw, int ld_raw, const float* mask_embed, int D, float logit_scale, const int* seg,
                    const float* scores, float temp, const int8_t* overlap, float alpha, float beta, int agg_add, const float* iou,
                    float fg_a, float fg_b, int mode, float* out, float* row_max, int* row_arg, int R, int C, void* stream);

/* ---- SAM box-prompted mask refinement (cfg.SAM.ENABLED: projects/HIPIE/hipie/hipie_img.py:241-246,367-390, models/sam.py; the
 * segment_anything 1.0 SamPredictor / MaskDecoder / TwoWayTransformer it runs).  The image encoder and every linear of the mask
 * decoder run on hipie_gemm / hipie_layernorm / hipie_attention(_tc); these cover the rest.
 * hipie_sam_attention: out[b, i, h*hd + d] = sum_j softmax_j(scale * q[qi(b), i, h] . k[ki(b), j, h]) v[ki(b), j, h][d], fp32 softmax.
 *   One side is short: Tq <= 32 (token self-attention T x T; token -> image, T queries over 4096 keys split over the lanes of a warp
 *   and combined) or else Tk <= 32 (image -> token, 4096 queries over T keys held in shared memory; 2 * Tk * H * hd * 4 B must stay
 *   <= 48 KB).  T = 5 output tokens + the sparse prompt tokens.  hd 16 or 32.  q / k / v fp32, head h at columns [h*hd, (h+1)*hd) of
 *   a row; rows q_ld / kv_ld apart, batches q_bs / kv_bs apart; q_index / kv_index (B) i32 or NULL map an output batch (a prompt) to
 *   its q / kv batch (an image: the layer-0 image stream is shared by every prompt of that image without a mask input).
 *   out_f32 and / or bf16 hi / lo planes (the A operand of out_proj), rows o_ld apart, batches o_bs apart.
 * hipie_sam_masks: x (N, h, w, 64) f32 = LayerNorm2d output of output_upscaling.0/1; w (64, 32, 2, 2) / bias (32) = output_upscaling.3;
 *   hyper (N, M, 32) = output_hypernetworks_mlps of M mask tokens (M = 1: mask 0, multimask_output=False; M = 3: masks 1..3).
 *   out (N, M, 2h, 2w) f32 = hyper[:, m] . GELU(ConvT(GELU(x))): the low-resolution logits, with the (N, 32, 2h, 2w) upscaled
 *   embedding never stored and computed once for all M masks.
 * hipie_sam_mask_embed: masks (N, 4 grid, 4 grid) f32 mask inputs; weights[10] = the device pointers of prompt_encoder.mask_downscaling
 *   .0.weight (4, 1, 2, 2), .0.bias, .1.weight, .1.bias (4), .3.weight (16, 4, 2, 2), .3.bias, .4.weight, .4.bias (16), .6.weight
 *   (256, 16, 1, 1), .6.bias (256) (the pointer array itself in host memory); LayerNorm2d eps; emb (B, grid^2, 256) f32 token-major
 *   image embeddings, img_index (N) i32 or NULL (identity) the image of each prompt.  src (N, grid^2, 256) f32 = emb[img(n)] +
 *   mask_downscaling(masks[n]) (Conv k2 s2 -> LayerNorm2d -> GELU -> Conv k2 s2 -> LayerNorm2d -> GELU -> Conv 1x1, GELU = erf form).
 * hipie_sam_postprocess: low (N, lh, lw) f32 logits -> per box n of image i = box_image[n], geom[i] = (h_in, w_in, h_large, w_large,
 *   height, width): bilinear to img_size^2 -> crop (h_in, w_in) -> bilinear to (h_large, w_large) -> > 0 (Sam.postprocess_masks,
 *   mask_threshold 0) -> area resize to (height, width) -> > 0.5 (hipie_img.py:385-386), uint8 at out + out_offset[n], row-major.
 *   max_pixels = the largest height * width.
 * hipie_sam_upscale: low (N, lh, lw) f32 logits of one image -> bilinear to img_size^2 -> crop (h_in, w_in) -> bilinear to (H, W)
 *   (SamPredictor.postprocess_masks, align_corners=False); out_f32 (N, H, W) the logits, or else out_u8 (N, H, W) = logit > threshold.
 * hipie_sam_mask_stats: the same chain for N <= 65535 masks of one crop (H, W = the crop size), reduced per mask without storing a
 *   pixel: stats (N, 8) i32 = (count(v > threshold + offset), count(v > threshold - offset), area = count(v > threshold), x0, y0, x1,
 *   y1, bands) -- the stability-score numerator and denominator and the inclusive box of the > threshold pixels ([0, 0, 0, 0] for an
 *   empty mask; segment_anything amg.py calculate_stability_score / batched_mask_to_box).  The thresholds are formed in double and
 *   compared in fp32, as segment_anything's Python sums against fp32 logits.  The last column counts the row bands merged.
 * hipie_sam_mask_emit: low (K, lh, lw) f32 logits, geom (K, 6) i32 device = (x0, y0, crop_h, crop_w, h_in, w_in) of each mask's crop
 *   of the (H, W) image: out (K, H, W) uint8 = the chain of hipie_sam_mask_stats at (y - y0, x - x0) > threshold inside the crop box, 0
 *   outside (amg.py uncrop_masks), pixel for pixel the evaluation the statistics counted. */
int hipie_sam_attention(const float* q, int64_t q_bs, int64_t q_ld, const int* q_index, const float* k, const float* v, int64_t kv_bs,
                        int64_t kv_ld, const int* kv_index, float* out_f32, void* out_hi, void* out_lo, int64_t o_bs, int64_t o_ld, int B,
                        int H, int Tq, int Tk, int hd, float scale, void* stream);
int hipie_sam_masks(const float* x, const float* w, const float* bias, const float* hyper, float* out, int N, int M, int h, int wd,
                    void* stream);
int hipie_sam_mask_embed(const float* masks, int N, const float* const* weights, float eps, const float* emb, const int* img_index,
                         int grid, float* src, void* stream);
int hipie_sam_postprocess(const float* low, int N, int lh, int lw, int img_size, const int* box_image, const int* geom,
                          const int64_t* out_offset, int64_t max_pixels, uint8_t* out, void* stream);
int hipie_sam_upscale(const float* low, int N, int lh, int lw, int img_size, int h_in, int w_in, int H, int W, float threshold,
                      float* out_f32, uint8_t* out_u8, void* stream);
int hipie_sam_mask_stats(const float* low, int N, int lh, int lw, int img_size, int h_in, int w_in, int H, int W, double threshold,
                         double offset, int* stats, void* stream);
int hipie_sam_mask_emit(const float* low, const int* geom, int K, int lh, int lw, int img_size, int H, int W, float threshold, uint8_t* out,
                        void* stream);

/* ---- hierarchical part segmentation (projects/HIPIE/hipie/demo_lib/part_segm_demo.py: PartSegmDemo, remap,
 * sem_to_instance_map_by_instances).
 * hipie_part_assign: sem (C, H, W) f32 class scores of the part vocabulary; group (C) i32 fine id -> coarse id, Cc = "no part" (entries
 *   outside 0..Cc are read as Cc); inst (N, H, W) uint8 instance masks (non-zero = inside).  fine (H, W) i32 = first index of the
 *   maximum over C (torch.argmax order: NaN wins, ties go to the lowest index); coarse (H, W) i32 = group[fine]; cnt_fine (N, C) and
 *   cnt_coarse (N, Cc + 1) i32 = per-instance pixel counts of each label (zeroed here).  N = 0 is valid (counts may then be NULL).
 * hipie_part_masks: labels (L, H, W) i32 label planes (fine and coarse), inst (N, H, W) uint8, pairs (P, 3) i32 = (plane, label,
 *   instance), plane < L and instance < N (validated by the caller): out (P, H, W) uint8 = (labels[plane] == label) & (inst[instance] != 0),
 *   so the masks of both levels leave in one launch. */
int hipie_part_assign(const float* sem, int C, int H, int W, const int* group, int Cc, const uint8_t* inst, int N, int* fine, int* coarse,
                      int* cnt_fine, int* cnt_coarse, void* stream);
int hipie_part_masks(const int* labels, int L, int H, int W, const uint8_t* inst, int N, const int* pairs, int P, uint8_t* out, void* stream);

/* ---- labelling SAM's automatic masks by voting against HIPIE's panoptic and part masks (projects/HIPIE/hipie/demo_lib/demo_utils.py:
 * vote, as driven by notebooks/Demo-HIPIE+SAM.ipynb).  The vote's map has channel 0 = 0.05f and channel m >= 1 = L_m(p) / (n(p) + 1e-5f),
 * n(p) = number of label planes covering p; its pooled sums are returned as exact uint64 fixed point (value * 2^32).  M <= 255,
 * H * W < 2^30.
 * hipie_label_cover: labels (M, H, W) uint8 (non-zero = inside; NULL when M = 0) -> bits (WD, H, W) u32 planar label bit sets, WD = 1 / 2 /
 *   4 / 8 for M <= 32 / 64 / 128 / 255 (bit m % 32 of word m / 32 = label plane m); sem_raw (H, W) i32 = argmax of the map (0 = background
 *   where no label covers p or where n(p) >= 20, else 1 + the first covering plane).
 * hipie_sam_vote: one chunk of Kc <= 64 masks (Kc, H, W) uint8, masks base .. base + Kc - 1 of K; bits from hipie_label_cover; labels
 *   >= first_part are part labels.  Adds, for each mask k of the chunk, acc[k, 0] += 0.05f * 2^32 * area, acc[k, 1 + m] += the fixed-point
 *   weights of its pixels inside plane m, area[k] += pixels, inter[k] += pixels covered by a part label (acc (K, M + 1), area / inter (K)
 *   u64, zeroed by the caller); raw (H, W) i32 (-1 = not yet covered, set by the caller) takes base + the first mask of the chunk covering
 *   p where it is still -1.  Chunks are launched in order on one stream. */
int hipie_label_cover(const uint8_t* labels, int M, int H, int W, uint32_t* bits, int* sem_raw, void* stream);
int hipie_sam_vote(const uint8_t* masks, int Kc, int H, int W, const uint32_t* bits, int M, int first_part, int base, int K,
                   unsigned long long* acc, unsigned long long* area, unsigned long long* inter, int* raw, void* stream);

/* ---- evaluation reductions (detectron2/evaluation/sem_seg_evaluation.py SemSegEvaluator.process; panopticapi
 * evaluation.py pq_compute_single_core as driven by COCOPanopticEvaluator).  Both accumulate with atomics on the given stream and do
 * not synchronise; invalid inputs are counted in *err (u64, accumulated, zeroed by the caller) and never binned.
 * hipie_semseg_confusion: sem (C, H, W) f32 class scores, gt (H, W) i32 labels: pred = the first index of the maximum over C
 *   (torch.argmax: NaN wins), g = C where gt == ignore_label, conf[pred * (C + 1) + g] += 1 into the (C + 1)^2 u64 matrix (rows =
 *   predictions, columns = GT).  GT labels outside 0..C-1 that are not ignore_label go to *err.  C <= 4096, H * W < 2^31.
 * hipie_panoptic_pairs: pred (H, W) i32 segment ids (0 = VOID, 1..S), gt_rgb (H, W, 3) uint8 the RGB-coded GT PNG (id = R + 256 G +
 *   65536 B), gt_ids (n_gt) i32 ascending ids listed in the image's segments_info: table[(n_gt + 2) x (S + 1)] u64 += pixel counts of
 *   (GT row, pred id), row 0 = GT VOID, rows 1..n_gt = gt_ids, row n_gt + 1 = GT ids in the PNG but not listed.  Predictions outside
 *   0..S go to *err.  n_gt <= 4096, S <= 65535, (n_gt + 2) (S + 1) <= 2^24. */
int hipie_semseg_confusion(const float* sem, int C, int H, int W, const int* gt, int ignore_label, unsigned long long* conf,
                           unsigned long long* err, void* stream);
int hipie_panoptic_pairs(const int* pred, const uint8_t* gt_rgb, int H, int W, const int* gt_ids, int n_gt, int S,
                         unsigned long long* table, unsigned long long* err, void* stream);

/* ---- instance mask overlaps (pycocotools maskApi.c rleIou on the RLEs of detectron2's COCOEvaluator).  One bit layout: a mask is its
 * row-major pixels (bit j of word w = pixel y * W + x = 32 w + j), zero-padded to whole 256-bit chunks, KW = hipie_mask_words(H, W) u32
 * words per mask.  N <= 1024 predictions, M <= 4096 GTs, H * W < 2^31; N = 0 / M = 0 launch nothing.  No call synchronises.
 * hipie_mask_pack: masks (N, H, W) uint8 (non-zero = inside) -> bits (N, KW), area[n] += pixel count (i32, zeroed by the caller).
 * hipie_rle_expand: GT g's column-major COCO runs (background first) as cumulative ends ends[offsets[g] .. offsets[g + 1]) (i32, offsets
 *   (M + 1) i64) -> bits (M, KW).  A list whose last end is not H * W is counted in *err (u64, accumulated).
 * hipie_mask_overlaps: inter (N, M) i32 (zeroed by the caller) += sum_k popc(pred_bits[n, k] & gt_bits[m, k]). */
int64_t hipie_mask_words(int H, int W);
int hipie_mask_pack(const uint8_t* masks, int N, int H, int W, uint32_t* bits, int* area, void* stream);
int hipie_rle_expand(const int* ends, const int64_t* offsets, int M, int H, int W, uint32_t* bits, unsigned long long* err, void* stream);
int hipie_mask_overlaps(const uint32_t* pred_bits, int N, const uint32_t* gt_bits, int M, int H, int W, int* inter, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* HIPIE_B200_H_ */
