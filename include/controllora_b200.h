/* controllora_b200 — C ABI of the H100-native ControlLoRA UNet hot path.
 *
 * The reference (HighCWu/ControlLoRA) is pure Python: its "FFI" for this path is the set of torch/ATen calls
 * issued by diffusers' UNet2DConditionModel and by models.py's attention processors.  Each entry point below
 * replaces one family of those calls; the reference call site it stands in for is cited (paths relative to
 * /root/reference, diffusers = the un-vendored diffusers 0.13/0.14 dependency).
 *
 * Conventions
 *   - every function is stream-ordered, takes raw device pointers + sizes, never allocates, never syncs,
 *     never throws; it returns 0 on success or a negative cl_status, with cl_last_error() giving the text.
 *   - activations are bf16, channels-last: an (N,H,W,C) image tensor and a (N*H*W, C) token matrix are the
 *     same memory.  Frozen weights are bf16, row-major [out, in] (conv: [out, ky, kx, in]).
 *   - trainable (LoRA / hint-encoder) parameters and all gradients of trainable parameters are fp32.
 *   - `stream` is a cudaStream_t passed as void* so that the header has no CUDA dependency.
 */
#ifndef CONTROLLORA_B200_H
#define CONTROLLORA_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
    CL_OK = 0,
    CL_ERR_INVALID = -1,   /* bad argument / unsupported shape */
    CL_ERR_CUDA = -2,      /* a CUDA runtime/driver call failed */
    CL_ERR_UNSUPPORTED = -3
} cl_status;

const char* cl_last_error(void);
int cl_version(void);
/* number of kernels this library has launched since load (bench.py's gpu_launches) */
int64_t cl_launch_count(void);

/* ------------------------------------------------------------------------------------------------------------
 * K1/K4: wgmma GEMM  D[M,N] = epilogue( A[M,K] * B[N,K]^T )   (bf16 x bf16 -> fp32 accumulators)
 *
 * Replaces: attn.to_q/to_k/to_v/to_out[0] + LoRALinearLayer side path  (models.py:124-147, 231-282, 373-423),
 *           diffusers FeedForward linears, Transformer2DModel proj_in/proj_out (1x1 conv == GEMM on NHWC),
 *           ResnetBlock2D conv1/conv2/conv_shortcut, Downsample2D/Upsample2D convs (3x3 as implicit GEMM),
 *           and their dX backward (same kernel on the transposed / flipped weight copies).
 *
 * a_mode 0: A is a row-major [M, K] matrix (lda elements between rows).
 * a_mode 1: A is an NHWC image (n_img, H, W, C); the GEMM row m = (n*H + h)*W + w reads the 3x3 window around
 *           (h, w) with zero padding 1; K = 9*C, k = (ky*3 + kx)*C + c.  B is [N, 9*C].   C % 64 == 0.
 * a_mode 2: as 1 but stride 2: output (n, ho, wo) of size (H/2, W/2) reads input (2ho+ky-pad_lo, 2wo+kx-pad_lo);
 *           pad_lo = 1 is diffusers' UNet Downsample2D(padding=1), pad_lo = 0 is the hint encoder's
 *           F.pad(0,1,0,1) + conv(padding=0) (models.py:591-598).
 *
 * LoRA epilogue (lora_up != NULL): `ext` is a bf16 [16, K] matrix appended below B's rows, so the tensor core also
 * produces e = A*ext^T (16 extra accumulator columns); t[j] = e[j] + e[j+8] (+ t_add[m, j]) for j < lora_rp and
 * D[m, n] += lora_scale * sum_j t[j] * lora_up[n*lora_rp + j].   (ext rows j / j+8 hold the bf16 hi / lo split of
 * LoRA-down row j, which keeps the rank-r path at ~fp32 accuracy like the reference's fp32 LoRALinearLayer.)
 * If t_out != NULL, t (fp32 [M, lora_rp]) is stored for the backward pass.
 * ---------------------------------------------------------------------------------------------------------- */
typedef struct {
    int32_t M, N, K;
    int32_t a_mode;
    const void* a;      /* bf16 */
    int64_t lda;        /* a_mode 0 only */
    int32_t n_img, H, W, C; /* a_mode 1/2: INPUT image geometry */
    int32_t pad_lo;     /* a_mode 2 */
    const void* b;      /* bf16 [N, K], row pitch ldb */
    int64_t ldb;
    const void* ext;    /* bf16 [16, K] row pitch ldb_ext, or NULL */
    int64_t ldb_ext;
    /* epilogue */
    const float* bias;       /* [N] or NULL */
    const float* row_bias;   /* [n_groups, >= N] (row pitch ld_row_bias, 0 = N) or NULL; group of row m = m / rows_per_group */
    int32_t rows_per_group;
    int64_t ld_row_bias;
    const void* residual;    /* bf16 [M, N] pitch ldr, or NULL; may alias out */
    int64_t ldr;
    const float* lora_up;    /* fp32 [N, lora_rp] or NULL */
    int32_t lora_rp;         /* 4 or 8 */
    float lora_scale;
    const float* t_add;      /* fp32 [M, lora_rp] or NULL */
    float* t_out;            /* fp32 [M, lora_rp] or NULL */
    void* out;               /* bf16 (out_fp32 = 0) or fp32 [M, N], pitch ldd */
    int64_t ldd;
    int32_t out_fp32;
    int32_t block_n;         /* 0 = auto */
    int32_t split_k;         /* <= 1: none.  > 1: K is cut into this many ranges, each CTA stores an fp32 partial tile
                                to split_ws and a second kernel sums them and applies bias / row_bias / residual
                                (deterministic: no atomics).  Not available with the LoRA epilogue. */
    void* split_ws;          /* device fp32 [split_k][M][N], required when split_k > 1 */
} cl_gemm_args;

int cl_gemm(const cl_gemm_args* args, void* stream);
/* Split count cl_gemm's heuristic recommends for these arguments (1 = none); size split_ws with it. */
int cl_gemm_split_hint(const cl_gemm_args* args);
/* The plan cl_gemm makes for these arguments, without launching: info[0] = tile width (block_n), info[1] = K splits,
   info[2] = CTAs per SM the kernel is launched for (1 or 2, chosen from the shape), info[3] = CTAs of that kernel the
   device keeps resident per SM at the shared-memory size of the launch (cudaOccupancyMaxActiveBlocksPerMultiprocessor). */
int cl_gemm_plan(const cl_gemm_args* args, int32_t info[4]);

/* ------------------------------------------------------------------------------------------------------------
 * K2: fused attention  O = softmax(Q K^T * scale) V  per (batch, head), probabilities never leave the SM.
 *
 * Replaces: attn.head_to_batch_dim + attn.get_attention_scores (baddbmm + softmax) + torch.bmm +
 *           attn.batch_to_head_dim   (models.py:126,137-142 / 244,267-272 / 381,404-409).
 * q/k/v/o: bf16 [B, N, H*d] token matrices with row strides ld* (elements); head h = columns [h*d, (h+1)*d).
 * lse (optional, fp32 [B, H, Nq]) receives log2-domain log-sum-exp of the scaled scores for the backward pass.
 * ---------------------------------------------------------------------------------------------------------- */
typedef struct {
    int32_t B, H, Nq, Nk, d;
    const void* q; int64_t ldq;
    const void* k; int64_t ldk;
    const void* v; int64_t ldv;
    void* o; int64_t ldo;
    float* lse;
    float scale;
} cl_attn_fwd_args;

int cl_attn_fwd(const cl_attn_fwd_args* args, void* stream);

/* Backward of cl_attn_fwd (what torch autograd derives for baddbmm/softmax/bmm in the reference): recomputes the
 * probabilities from q, k and `lse`.  `delta` is fp32 scratch [B, H, Nq].  dq and/or (dk, dv) may be NULL to skip
 * them (e.g. cross-attention to the frozen text encoder needs no dk/dv when its k/v projections carry no LoRA). */
typedef struct {
    int32_t B, H, Nq, Nk, d;
    const void* q; int64_t ldq;
    const void* k; int64_t ldk;
    const void* v; int64_t ldv;
    const void* o; int64_t ldo;
    const void* d_o; int64_t lddo;
    const float* lse;
    float* delta;
    void* dq; int64_t lddq;
    void* dk; int64_t lddk;
    void* dv; int64_t lddv;
    float scale;
} cl_attn_bwd_args;

int cl_attn_bwd(const cl_attn_bwd_args* args, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * K5: normalisation.  GroupNorm(+SiLU) on NHWC [n, HW, C] and LayerNorm on [T, C], forward and dX backward.
 * Replaces torch.nn.GroupNorm / F.silu / LayerNorm inside diffusers ResnetBlock2D, Transformer2DModel,
 * BasicTransformerBlock, UNet conv_norm_out, and models.py:515-543 (ConvBlock2D, where dgamma/dbeta are needed).
 * GroupNorm is one kernel launch per direction and needs no scratch; `stats` (fp32 [n, G, 2] = mean, rstd) feeds the
 * backward.
 * ---------------------------------------------------------------------------------------------------------- */
int cl_groupnorm_fwd(const void* x, const float* gamma, const float* beta, void* y, float* stats,
                     int n, int HW, int C, int G, float eps, int silu, void* stream);
int cl_groupnorm_bwd(const void* x, const void* dy, const float* gamma, const float* beta, const float* stats,
                     void* dx, float* dgamma /* nullable, accumulated */, float* dbeta, int n, int HW,
                     int C, int G, int silu, int accumulate_dx, void* stream);
int cl_layernorm_fwd(const void* x, const float* gamma, const float* beta, void* y, float* stats /* [T,2] */,
                     int T, int C, float eps, void* stream);
int cl_layernorm_bwd(const void* x, const void* dy, const float* gamma, const float* stats, void* dx, int T, int C,
                     int accumulate_dx, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Elementwise glue (bf16, channels-last).  GEGLU = diffusers FeedForward's `a * gelu(g)` on p = [a | g].
 * ---------------------------------------------------------------------------------------------------------- */
int cl_geglu_fwd(const void* p, void* out, int64_t T, int F, void* stream);
int cl_geglu_bwd(const void* p, const void* dout, void* dp, int64_t T, int F, void* stream);
int cl_add(const void* a, const void* b, void* out, int64_t n, void* stream);
int cl_upsample2x_fwd(const void* x, void* y, int n, int H, int W, int C, void* stream);      /* F.interpolate nearest */
int cl_upsample2x_bwd(const void* dy, void* dx, int n, int H, int W, int C, int accumulate, void* stream);
int cl_zero_insert2x(const void* x, void* y, int n, int H, int W, int C, int off, void* stream); /* stride-2 adjoint */
int cl_concat_channels(const void* a, const void* b, void* out, int64_t M, int Ca, int Cb, void* stream); /* torch.cat(dim=1) */
int cl_slice_channels(const void* src, void* dst, int64_t M, int Cs, int c_off, int Cd, int accumulate, void* stream);
int cl_nchw_to_nhwc(const void* x, int x_is_fp32, void* y, int n, int C, int HW, void* stream);
int cl_nhwc_to_nchw_f32(const void* x, float* y, int n, int C, int HW, int accumulate, void* stream);
int cl_f32_to_bf16(const float* x, void* y, int64_t n, void* stream);
int cl_bf16_to_f32(const void* x, float* y, int64_t n, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * UNet edges: conv_in (NCHW fp32 -> NHWC bf16), conv_out (NHWC bf16 -> NCHW fp32) + its dX, sinusoidal timestep
 * embedding, tiny-M linear (time MLP and all ResnetBlock2D.time_emb_proj at once), fused MSE loss + gradient
 * (train_text_to_image_control_lora.py:782-783).
 * ---------------------------------------------------------------------------------------------------------- */
int cl_conv_in(const float* x, const void* w /* bf16 [Cout][3][3][Cin] */, const float* bias, void* y, int n, int Cin,
               int H, int W, int Cout, void* stream);
int cl_conv_out(const void* x, const void* w /* bf16 [4][3][3][C] */, const float* bias, float* y, int n, int H, int W,
                int C, int Cout, void* stream);
int cl_conv_out_bwd(const float* dy, const void* w, void* dx, int n, int H, int W, int C, int Cout, void* stream);
int cl_timestep_embedding(const float* t, float* out, int B, int dim, void* stream);
int cl_small_linear(const float* x, const void* w, const float* bias, float* out, int Bt, int N, int K, int silu_in,
                    int silu_out, void* stream);
int cl_mse_loss(const float* pred, const float* target, float* loss, float* dpred, int64_t n, float gscale, void* stream);
/* Step glue in front of the UNet (replaces train_text_to_image_control_lora.py:757-765 `torch.randn_like` / `torch.randint` /
 * `noise_scheduler.add_noise` and :774-779 target selection): Philox4x32-10 noise + one timestep per image, counter-based
 * on (seed, *step_counter); *step_counter is advanced by one on the stream (CUDA-graph safe).  x0 / noisy / target:
 * [B, per_image] fp32 (per_image % 4 == 0); sqrt_ac / sqrt_1mac: device tables [num_train_timesteps]; timesteps: [B] fp32. */
int cl_add_noise(const float* x0, const float* sqrt_ac, const float* sqrt_1mac, unsigned long long* step_counter,
                 unsigned long long seed, int num_train_timesteps, int v_prediction, float* noisy, float* target,
                 float* timesteps, int B, int per_image, void* stream);
/* classifier-free-guidance combine + DDIM (eta = 0) update of the denoise loop, one fused elementwise kernel:
 * eps2 = [uncond | cond] noise predictions (each n_half floats), latents updated in place. */
/* VAE (train_text_to_image_control_lora.py:753-754, pipeline decode): row softmax of the one-head AttentionBlock
 * (p = softmax(scale * s) per row, fp32 in, bf16 out, cols % 4 == 0, <= 12288) and the post_quant_conv bias as a per-channel
 * shift of NCHW fp32 latents (y = mul * x + shift[c]). */
int cl_softmax_rows(const float* s, void* p, int rows, int cols, float scale, void* stream);
/* CLIP text encoder (transformers CLIPTextModel, train_text_to_image_control_lora.py:768 `text_encoder(batch["input_ids"])[0]`):
 * token + position embedding gather (bf16 tables, ids int64 [rows], row r is position r % T), the in-place quick_gelu
 * x * sigmoid(1.702 x) of CLIPMLP, and the causal self-attention of the 77-token sequence (T <= 128, head dim <= 64; fp32
 * online softmax, one CTA per (batch, head)); qkv [B*T, 3*heads*d] bf16 = q | k | v, out [B*T, heads*d] bf16. */
int cl_clip_embed(const int64_t* ids, const void* tok, const void* pos, void* out, int rows, int T, int C, int vocab, void* stream);
int cl_quick_gelu(void* x, int64_t n, void* stream);
int cl_causal_attention_small(const void* qkv, void* out, int B, int T, int heads, int d, float scale, void* stream);
int cl_channel_affine_nchw(const float* x, float* y, const float* shift, float mul, int n, int C, int64_t hw, void* stream);
/* strided weight-space helpers of the dense (concat_hidden, models.py:208-214) control MLP: bf16 view / transpose of an fp32
 * master (dst[i*ld + j] = bf16(alpha * src[i*s_i + j*s_j])) and strided fp32 accumulation (dst[i*ld + j] += alpha * src[i*J + j]) */
int cl_cast_matrix_bf16(const float* src, int64_t s_i, int64_t s_j, void* dst, int64_t ld, int I, int J, float alpha, void* stream);
int cl_axpy_matrix_f32(const float* src, float* dst, int64_t ld, int I, int J, float alpha, void* stream);
int cl_cfg_ddim_step(const float* eps2, float* latents, int64_t n_half, float guidance, float sqrt_at, float sqrt_1m_at,
                     float sqrt_aprev, float sqrt_1m_aprev, void* stream);
/* CFG + DPM-Solver++(2M) update (diffusers DPMSolverMultistepScheduler defaults; the scheduler of the reference's
 * validation loop / apps): x0 = (x - sigma_s eps)/alpha_s; x <- c_x x + c_m0 x0 + c_m1 x0_prev; x0_prev <- x0.        */
int cl_cfg_dpmpp_step(const float* eps2 /* [2B,...] = [uncond | cond] */, float* latents, float* x0_prev, int64_t n_half,
                      float guidance, float alpha_s, float sigma_s, float c_x, float c_m0, float c_m1, void* stream);
/* Graph-replayable form of the two loops above: per-step scalars come from device tables indexed by *step_ctr.
 * cl_sampler_prep: x2 = [latents | latents], tt[0..B2) = ts_table[*step_ctr].
 * cl_cfg_solver_step_dev: kind 0 = DDIM (coef row: sqrt_at, sqrt_1m_at, sqrt_aprev, sqrt_1m_aprev), kind 1 =
 *   DPM-Solver++(2M) (alpha_s, sigma_s, c_x, c_m0, c_m1); coef is [num_steps][8] fp32; then *step_ctr += 1 on the stream. */
int cl_sampler_prep(const float* latents, float* x2, float* tt, const float* ts_table, const unsigned long long* step_ctr,
                    int64_t n_half, int B2, void* stream);
int cl_cfg_solver_step_dev(const float* eps2, float* latents, float* x0_prev, const float* coef, unsigned long long* step_ctr,
                           int64_t n_half, float guidance, int kind, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * LoRA side path (diffusers LoRALinearLayer instances created at models.py:89-97,185,316-323).
 *
 * cl_lora_pack_batch: one launch converts every fp32 LoRA master weight of a step into the operands the fused GEMM
 *   consumes (kind 0: bf16 hi/lo `ext` rows; kind 1: fp32 [N, rp] `lora_up` table).  `descs` lives in device memory.
 * cl_skinny_atb:   out[j*so_j + c*so_c] += alpha * sum_m a[m*lda + j] * b[m*ldb + c]      (dA / dB reductions)
 * cl_rowdot:       e[m*rp + j] = sum_n a[m*lda + n] * u[n*rp + j]                         (dY * B_up when no dX GEMM runs)
 * cl_rowmat:       out[m, i] (+)= alpha * sum_j a[m*lda + j] * w[i*sw_i + j*sw_j]         (rank-r x rank-r per-row maps)
 * cl_skinny_small: out[i*J + j] += alpha * sum_m a[m*lda + i] * b[m*ldb + j]
 * cl_small_matmul: weight-space fp32 product with arbitrary strides.
 * ---------------------------------------------------------------------------------------------------------- */
typedef struct {
    const void* src;   /* fp32 */
    void* dst;
    int32_t kind;      /* 0: ext (bf16 [16, ld] hi/lo rows), 1: table (fp32 [K, ld]), 2: bf16 [K, ld] table, value in hi and lo slots */
    int32_t r, K;      /* src(j, k), j < r, k < K */
    int64_t s_j, s_k;  /* element strides of src */
    int32_t ld;        /* dst leading dimension (elements) */
    int32_t row_off;   /* first ext row / table column written */
    float mul;         /* factor applied to every packed value (1/scale for the unscaled stacked-value quirk, models.py:260,265,397,402) */
    int32_t pad_;
} cl_pack_desc;

int cl_lora_pack_batch(const cl_pack_desc* descs_dev, int n_desc, int max_elems, void* stream);
int cl_skinny_atb(const float* a, int lda, int r, const void* b, int64_t ldb, float* out, int64_t so_j, int64_t so_c,
                  float alpha, int M, int C, void* stream);
/* batched form: up to CL_SKINNY_MAX independent skinny reductions in one launch (descs is a HOST array, passed by value) */
#define CL_SKINNY_MAX 16
typedef struct {
    const float* a; int32_t lda; int32_t r;   /* fp32 [M, lda], first r (<= 8) columns used */
    const void* b; int64_t ldb;               /* bf16 [M, ldb], C columns */
    float* out; int64_t so_j, so_c;           /* out[j*so_j + c*so_c] += ... */
    float alpha; int32_t M, C;
} cl_skinny_desc;
int cl_skinny_atb_batch(const cl_skinny_desc* descs, int n, void* stream);
int cl_rowdot(const void* a, int64_t lda, const float* u, int rp, float* e, int M, int N, void* stream);
int cl_rowmat(const float* a, int lda, const float* w, int sw_i, int sw_j, int I, int J, float alpha, void* out, int ldo,
              int out_mode, int col_off, int lo_off, int accumulate, int M, void* stream);
int cl_hilo_combine(const float* src, float* dst, int64_t M, int nb, void* stream);  /* [M,16nb] hi|lo blocks -> [M,8nb] */
int cl_rank_update(const void* x, const float* t, int ldt, const float* tab, int rp, float alpha, void* out, int64_t M,
                   int C, void* stream);
/* V2 control injection (models.py:369, 415:  h' = h + s * up(down([h ; c]))) fused around the rank-4 update:
 *   fwd: t = hi/lo-combine(th16 [M,16]) + uc [M, rc<=4];  out = x + alpha * t[:, :4] tab^T (tab fp32 [C, 4]);  t_out [M, 8] kept
 *   bwd: dt [M, 4] = dy * up (fp32 [C, 4]);  dh = dy + alpha * dt * down^T (fp32 [C, 4]; dh nullable)                      */
int cl_v2_inject_fwd(const void* x, const float* th16, const float* uc /* nullable */, int ldu, int rc, const float* tab,
                     float alpha, void* out, float* t_out, int64_t M, int C, void* stream);
int cl_v2_inject_bwd(const void* dy, const float* up, const float* down, float alpha, float* dt_out, void* dh /* nullable */,
                     int M, int C, void* stream);
/* One pass "project, add, update" (the V2 forward without a separate skinny GEMM):
 *   t [M, 4] = x * proj (fp32 [C, 4]) (+ uc [M, rc]);   y = x + alpha * t * upd^T (fp32 [C, 4]).                            */
int cl_rank4_project_update(const void* x, const float* proj, const float* upd, const float* uc /* nullable */, int ldu, int rc,
                            float alpha, float* t_out, void* y, int M, int C, void* stream);                                            /* out = x + alpha * t * tab^T */
int cl_skinny_small(const float* a, int lda, int I, const float* b, int ldb, int J, float* out, float alpha, int M,
                    void* stream);
int cl_small_matmul(const float* a, int64_t sa_i, int64_t sa_j, const float* b, int64_t sb_j, int64_t sb_k, float* out,
                    int64_t so_i, int64_t so_k, int I, int J, int K, float alpha, int accumulate, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * K6: hint-encoder training support (the ControlLoRA conv stack of models.py:434-835 is trainable, so unlike the UNet
 * it needs weight gradients and a per-step re-layout of its fp32 master weights).
 *   cl_conv_wgrad:       dW[co,ci,ky,kx] += alpha * sum dY * X(shifted)   on wgmma (MN-major operands, split-K + RED)
 *   cl_conv_weight_prep: w fp32 [Cout][Cin][k][k] -> wf bf16 [Cout][k*k][Cin] (forward) and wd bf16 [Cin][k*k flipped][Cout] (dX)
 *   cl_colsum:           out[c] += alpha * sum_m x[m, c]                  (bias gradients)
 *   cl_conv_in_wgrad:    weight gradient of the 3-channel conv_in (SIMT)
 * ---------------------------------------------------------------------------------------------------------- */
int cl_conv_wgrad(const void* dy, const void* x, float* dw, int n_img, int H, int W, int Cin, int Cout, int ksize, int stride,
                  int pad_lo, float alpha, void* stream);
int cl_conv_weight_prep(const float* w, void* wf, void* wd /* nullable */, int Cout, int Cin, int ksize, void* stream);
int cl_colsum(const void* x, float* out, int64_t M, int C, float alpha, void* stream);
int cl_conv_in_wgrad(const float* x, const void* dy, float* dw, int n, int Cin, int H, int W, int Cout, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * K8: optimizer on the flat fp32 parameter / gradient arenas (train_text_to_image_control_lora.py:791-796:
 * clip_grad_norm_(max_norm) + torch.optim.AdamW step + zero_grad), no host synchronisation.
 *   cl_sumsq:  *out += sum x^2   (call once per arena after zeroing *out; the total grad norm)
 *   cl_adamw:  g' = g * grad_scale * min(1, max_norm / (sqrt(*gnorm_sq) * grad_scale + 1e-6));  AdamW(p, g', m, v);  g = 0
 * ---------------------------------------------------------------------------------------------------------- */
int cl_sumsq(const float* x, int64_t n, float* out, void* stream);
int cl_adamw(float* p, float* g, float* m, float* v, int64_t n, float lr, float beta1, float beta2, float eps,
             float weight_decay, int step, const float* gnorm_sq, float max_norm, float grad_scale, int zero_grad,
             void* stream);
/* the same optimizer tail for a CUDA-graph-captured step: cl_step_begin clears the squared-norm accumulator and advances a
 * device-side step counter, cl_adamw_dev takes its bias corrections from that counter (train_...:791-796 without a host scalar) */
int cl_step_begin(float* gnorm_sq, int64_t* step_dev, void* stream);
int cl_adamw_dev(float* p, float* g, float* m, float* v, int64_t n, float lr, float beta1, float beta2, float eps,
                 float weight_decay, const int64_t* step_dev, const float* gnorm_sq, float max_norm, float grad_scale,
                 int zero_grad, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Canny annotator: cv2.Canny(img, lo, hi) (aperture 3, L2gradient = false) bit for bit, and the float32 tensors the
 * reference builds from it.  Replaces the OpenCV call and its arithmetic at process/diffusiondb_canny.py:35-45 (dataset of
 * tasks/train_canny_v2.py: pixel_values = img / 127.5 - 1, guide = canny / 127.5 - 1 repeated to 3 channels),
 * apps/gradio_canny2image.py:71-74 (apply_canny + HWC3 + [..., ::-1] / 127.5 - 1) and annotator/canny/__init__.py:6
 * (CannyDetector, also used by tasks/make_dataset_diffusiondb_2m_first_5k_canny.py:27).
 *   img:        uint8 NHWC [B, H, W, C], C = 1 or 3, channels used in the order given (a tie in gradient magnitude goes
 *               to the first channel, so RGB and BGR input can differ); B*H*W < 2^31.
 *   thresholds: device fp32 [B, 2] (lo, hi) per image, read on the device (swapped when lo > hi, then floored), so a
 *               captured graph can replay with new values.
 *   labels:     device int32 scratch [B*H*W].
 *   outputs (any non-empty subset, NULL = skip): edges uint8 [B, H, W] (0 / 255); guide fp32 NCHW [B, 3, H, W] (+-1.0);
 *               pixels fp32 NCHW [B, 3, H, W] = img / 127.5 - 1 with both operations rounded to fp32 (C = 3 only).
 * Four launches whatever the data (union-find hysteresis), no host synchronisation.
 * ---------------------------------------------------------------------------------------------------------- */
int cl_canny(const uint8_t* img, int B, int H, int W, int C, const float* thresholds, int32_t* labels, uint8_t* edges,
             float* guide, float* pixels, void* stream);

#ifdef __cplusplus
}
#endif
#endif
