/* vxb200.h -- C ABI of libvxb200.so: hand-written sm_90a kernels for the V-Express denoising hot path.
 *
 * The reference (tencent-ailab/V-Express) is 100% Python and has no FFI: every arithmetic call on this path is a
 * torch / diffusers library call.  Each entry point below replaces one family of those call sites (cited as
 * reference file:line, relative to the upstream repo) and is what a Python binding of the reference would
 * load with ctypes (INTEGRATION.md shows the stub).  Conventions:
 *   - all pointers are DEVICE pointers unless stated; activations are bf16, row-major token matrices
 *     [rows, C] with rows = ((b f) h w) ("channels-last"); `ld*` are row strides in ELEMENTS;
 *   - weights are bf16 [N, K] (nn.Linear layout; 3x3 conv weights repacked to [Cout, (ky kx cin)]);
 *     biases / norm affine parameters are fp32;
 *   - `stream` is a cudaStream_t; calls are asynchronous, re-entrant, CUDA-graph capturable;
 *   - return value 0 = success; otherwise vx_last_error() holds a message (thread-local).  Nothing is
 *     swallowed and there is no CPU fallback.
 */
#ifndef VXH100_H
#define VXH100_H
#ifdef __cplusplus
extern "C" {
#endif

const char* vx_last_error(void);
int vx_abi_version(void);
int vx_require_sm90(void); /* fails unless the current device is sm_90 (H100) */

/* ---- wgmma + TMA GEMM: out = (concat_K(A, A2) @ W^T + bias + bias2[row / bias2_div]) * scale + residual.
 * Replaces nn.Linear / 1x1 nn.Conv2d: diffusers Attention.to_q/to_k/to_v/to_out (modules/attention.py:321-360,
 * modules/motion_module.py:280-290), FeedForward (attention.py:375, motion_module.py:233), proj_in/proj_out
 * (modules/transformer_3d.py:64-66,93-95; motion_module.py:122,144), conv_shortcut (modules/resnet.py:213-215).
 * A2 != NULL folds torch.cat([h, skip], 1) (modules/unet_3d_blocks.py:694,831) into the K loop.
 * out_f32 = 1 stores fp32 (attention scores of the VAE mid block). block_n = 0 lets the library choose. */
int vx_gemm_bf16(const void* A, long long lda, int K1, const void* A2, long long lda2, int K2, const void* W,
                 long long ldw, int M, int N, const float* bias, const float* bias2, int bias2_div, float scale,
                 const void* residual, long long ldr, void* out, long long ldc, int out_f32, int block_n,
                 void* stream);

/* ---- e4m3 wgmma GEMM (opt-in FP8 mode, UNet3DConditionModel.enable_fp8_linear): A [M, K] and W [N, K] hold
 * float8_e4m3fn codes (K-major; K, lda, ldw multiples of 16) with one fp32 scale per row of A (a_scale, from
 * vx_layernorm_fp8) and per output channel of W (w_scale, ops.quantize_fp8_weight).  out = epilogue(a_scale[m] *
 * w_scale[n] * sum_k A[m,k] W[n,k]) in bf16, the epilogue (bias, bias2, scale, residual; or geglu = 1 with W, w_scale and
 * bias packed per column tile as for vx_gemm_bf16) as in vx_gemm_bf16.  Replaces the nn.Linear layers fed by an
 * nn.LayerNorm: the fused attn1 to_q|to_k|to_v, attn1_5.to_q, attn2.to_q and ff.net.0.proj (GEGLU) of the spatial
 * transformer blocks (modules/attention.py:329-375) and the fused to_q|to_k|to_v and ff.net.0.proj of the motion modules
 * (modules/motion_module.py:228-234,280-290).  block_n = 0 lets the library choose. */
int vx_gemm_fp8(const void* A, long long lda, const float* a_scale, int K, const void* W, long long ldw,
                const float* w_scale, int M, int N, const float* bias, const float* bias2, int bias2_div, float scale,
                const void* residual, long long ldr, void* out, long long ldc, int geglu, int block_n, void* stream);

/* ---- LayerNorm folded into the consumer GEMM (VX_LN_FOLD=1; run on hardware in round 2: parity green, no gain with the
 * separate statistics pass -- see vx_gemm_rowsums_bf16 for the variant without one).  vx_row_stats writes (mean, rstd) per row of the
 * un-normalised activations; vx_gemm_lnfold_bf16 computes rstd[m] * (A @ Wt^T - mean[m] * colsum) + bias with
 * Wt = W * gamma, colsum[n] = sum_k Wt[n,k], bias[n] = sum_k beta[k] W[n,k] + b[n]: the nn.LayerNorm + nn.Linear pairs
 * of modules/attention.py:329-375 and modules/motion_module.py:228-234 without writing LayerNorm(x) to HBM. */
int vx_row_stats(const void* x, long long ldx, long long rows, int C, float eps, float* stats, void* stream);
int vx_gemm_lnfold_bf16(const void* A, long long lda, int K, const void* Wt, long long ldw, int M, int N,
                        const float* stats, const float* colsum, const float* bias, const float* bias2, int bias2_div,
                        float scale, const void* residual, long long ldr, void* out, long long ldc, int geglu,
                        int block_n, void* stream);

/* LayerNorm statistics handed from GEMM to GEMM.  Every nn.LayerNorm of the transformer blocks normalises the output of a
 * Linear (+ residual) -- attn.to_out / proj_in of modules/attention.py:321-375, modules/transformer_3d.py:64-66,
 * modules/motion_module.py:122,228-234,300-321 -- and feeds another Linear.  vx_gemm_rowsums_bf16 is vx_gemm_bf16 (linear
 * epilogue, bf16 out) that also writes per output row `*nparts` = 2 * ceil(N / block_n) float2 partials (sum, sum of
 * squares) of the ROUNDED outputs, row_parts[slot * parts_stride + m] (parts_cap slots allocated); vx_gemm_lnparts_bf16 is vx_gemm_lnfold_bf16 that
 * derives mean / rstd from such partials (slot order, fp32, variance = E[x^2] - mean^2, eps as nn.LayerNorm).  Together:
 * LayerNorm(x) @ W^T with neither a normalisation pass nor a statistics pass over x. */
int vx_gemm_rowsums_bf16(const void* A, long long lda, int K1, const void* A2, long long lda2, int K2, const void* W,
                         long long ldw, int M, int N, const float* bias, const float* bias2, int bias2_div, float scale,
                         const void* residual, long long ldr, void* out, long long ldc, int block_n, float* row_parts,
                         long long parts_stride, int parts_cap, int* nparts, void* stream);
int vx_gemm_lnparts_bf16(const void* A, long long lda, int K, const void* Wt, long long ldw, int M, int N,
                         const float* row_parts, long long parts_stride, int nparts, float eps, const float* colsum,
                         const float* bias, const float* bias2, int bias2_div, float scale, const void* residual,
                         long long ldr, void* out, long long ldc, int geglu, int block_n, void* stream);

/* nn.LayerNorm -> nn.Linear in ONE kernel for K <= 512 (the UNet's 320-wide level): same folded parameters as
 * vx_gemm_lnfold_bf16, but the (mean, rstd) of a row tile are computed inside the kernel from the shared-memory resident
 * 128 x K tile of A (two-pass variance, eps as nn.LayerNorm), which also serves every column tile of that row tile, so
 * only W streams through the TMA ring.  Neither LayerNorm(A) nor a statistics array is written to HBM.  Replaces the
 * norm1/norm1_5/norm2/norm3 -> to_q/to_k/to_v/ff.net.0 pairs of modules/attention.py:329-375 and the norms -> qkv / ff_norm
 * -> ff pairs of modules/motion_module.py:228-234,300-321 at K = 320. */
int vx_gemm_ln_bf16(const void* A, long long lda, int K, const void* Wt, long long ldw, int M, int N,
                    const float* colsum, const float* bias, float eps, const float* bias2, int bias2_div, float scale,
                    const void* residual, long long ldr, void* out, long long ldc, int geglu, int block_n, void* stream);

/* ---- wgmma implicit-GEMM 3x3 convolution, stride 1, pad 1, NHWC.  X [NB,H,W,C]; W [Cout, 9*C].
 * Replaces InflatedConv3d / nn.Conv2d 3x3 (modules/resnet.py:9-17,165-167,194-196; Upsample3D conv :51) and the
 * VAE decoder convs (diffusers AutoencoderKL, SURVEY.md B.6).  bias2 = per-sample bias (time embedding,
 * modules/resnet.py:225-236), residual = the resnet skip (:246-249). */
int vx_conv3x3_bf16(const void* X, int NB, int H, int W, int C, const void* Wt, int Cout, const float* bias,
                    const float* bias2, int bias2_div, float scale, const void* residual, long long ldr, void* out,
                    long long ldc, int block_n, void* stream);

/* ---- wgmma flash attention (no mask): q [Bq*Nq, ldq], k/v [Bkv*Nk, ld], out [Bq*Nq, ldo]; heads*hd columns;
 * kv batch of query batch b is b / kv_div.  Replaces F.scaled_dot_product_attention inside AttnProcessor2_0 for
 * attn1 (modules/mutual_self_attention.py:176-186) and attn1_5 (:202-219, kv_div = frames per window). */
int vx_flash_attention(const void* q, long long ldq, const void* k, long long ldk, const void* v, long long ldv,
                       void* out, long long ldo, int Bq, int Nq, int Bkv, int Nk, int heads, int hd, int kv_div,
                       void* stream);

/* ---- temporal self-attention over the f frames of a window for every (b, pixel, head); q/k/v are column slices
 * of one [(b f hw), ld] matrix.  Replaces VersatileAttention.forward incl. both rearranges
 * (modules/motion_module.py:351-388). */
int vx_temporal_attention(const void* q, const void* k, const void* v, long long ld, void* out, long long ldo, int b,
                          int f, int HW, int heads, int hd, void* stream);

/* ---- attention of every query row to the Lk (<= 8) tokens of its frame: audio cross-attention attn2
 * (modules/mutual_self_attention.py:229-242).  k/v rows = frame*Lk + token. */
int vx_smallkv_attention(const void* q, long long ldq, const void* k, const void* v, long long ldkv, void* out,
                         long long ldo, long long rows, int rows_per_frame, int heads, int hd, int Lk, void* stream);

/* ---- per-frame GroupNorm (+SiLU) of the channel concatenation [x1 | x2] (x2 may be NULL), two deterministic
 * kernels.  Replaces InflatedGroupNorm / nn.GroupNorm + F.silu (modules/resnet.py:20-28,220-221,235-241;
 * modules/transformer_3d.py:124; modules/motion_module.py:156; modules/unet_3d.py:571-572).
 * partial: float[vx_groupnorm_stats_ws_floats(NB, G, S)] workspace shared by the two calls. */
int vx_groupnorm_stats_ws_floats(int NB, int G, int S);
int vx_groupnorm_stats(const void* x1, long long ld1, int C1, const void* x2, long long ld2, int C2, int NB, int HW,
                       int G, int S, float* partial, void* stream);
int vx_groupnorm_apply(const void* x1, long long ld1, int C1, const void* x2, long long ld2, int C2, int NB, int HW,
                       int G, int S, const float* partial, const float* gamma, const float* beta, float eps,
                       int silu, void* out, long long ldo, void* stream);
/* Number of GroupNorm CTAs (for C channels) resident at once on the device: NB * S must not exceed it for the fused kernel. */
int vx_groupnorm_capacity(int C);
/* Both passes in ONE launch behind a per-frame rendezvous (the second read of a frame is served by the L2 at UNet sizes).
 * counters: int[2*NB], zeroed once by the caller (the kernel recycles them).  Returns 2 without launching when NB*S CTAs
 * cannot be co-resident: use the two-kernel pair then.  Results are bit-identical to vx_groupnorm_stats + _apply. */
int vx_groupnorm_fused(const void* x1, long long ld1, int C1, const void* x2, long long ld2, int C2, int NB, int HW, int G,
                       int S, float* partial, int* counters, const float* gamma, const float* beta, float eps, int silu,
                       void* out, long long ldo, void* stream);

/* GroupNorm of small frames (the 8x8 / 16x16 levels) with the frame resident in the shared memory of a thread-block
 * cluster: one pass over HBM, partial statistics exchanged through distributed shared memory, no workspace.  Same
 * operands as vx_groupnorm_fused; returns 2 without launching when the frame does not fit a cluster of <= 8 CTAs. */
int vx_groupnorm_cluster(const void* x1, long long ld1, int C1, const void* x2, long long ld2, int C2, int NB, int HW,
                         int G, const float* gamma, const float* beta, float eps, int silu, void* out, long long ldo,
                         void* stream);

/* ---- LayerNorm over C, optional + pe[(row / rows_per_frame) % pe_frames] (temporal positional encoding).
 * Replaces nn.LayerNorm (modules/attention.py:329-333; modules/motion_module.py:228,234) and
 * PositionalEncoding.forward (modules/motion_module.py:275-277). */
int vx_layernorm(const void* x, long long ldx, long long rows, int C, const float* gamma, const float* beta,
                 float eps, const float* pe, int rows_per_frame, int pe_frames, void* out, long long ldo,
                 void* stream);
/* vx_layernorm writing the A operand of vx_gemm_fp8: out [rows, ldo] float8_e4m3fn codes sat_rn(y / row_scale[row]) of
 * the fp32 LayerNorm (+ pe) result y (not rounded through bf16), row_scale[row] = amax(|y|) / 448 (1 for an all-zero
 * row).  Same call sites as vx_layernorm, for the LayerNorms that feed the GEMMs listed at vx_gemm_fp8. */
int vx_layernorm_fp8(const void* x, long long ldx, long long rows, int C, const float* gamma, const float* beta,
                     float eps, const float* pe, int rows_per_frame, int pe_frames, void* out, long long ldo,
                     float* row_scale, void* stream);

/* ---- GEGLU gate: x [rows, 2*inner] = (h | gate) -> h * gelu_erf(gate) (diffusers GEGLU, SURVEY.md B.3). */
int vx_geglu(const void* x, long long ldx, long long rows, int inner, void* out, long long ldo, void* stream);

/* ---- row softmax of fp32 scores -> bf16 (VAE mid-block single-head attention, SURVEY.md B.6). */
int vx_softmax_rows(const float* x, long long ldx, long long rows, int n, void* out, long long ldo, void* stream);

/* ---- conv_in: 3x3 conv from planar (n,c,h,w) bf16 with Cin <= 8 to NHWC, + bias + gathered NHWC addend
 * (kps_features, modules/unet_3d.py:485-487); optional per-pixel pre-transform bf16(pre_w @ bf16(pre_scale*v) + pre_b)
 * (latents / 0.18215 and the VAE post_quant_conv, pipelines/v_express_pipeline.py:155,159). w fp32 [Cin*9, Cout]
 * (transposed), Cin = 4. */
int vx_conv_in(const void* in, long long sn, long long sc, int NB, int H, int W, int Cin, int Cout, const float* w,
               const float* bias, const void* addend, const int* add_frame, long long add_ld, float pre_scale,
               const float* pre_w, const float* pre_b, void* out, long long ldo, void* stream);

/* ---- conv_out: 3x3 conv from NHWC bf16 to Cout <= 4 planar output (modules/unet_3d.py:573; VAE conv_out);
 * post = 1 applies (v/2 + 0.5).clamp(0,1) (pipelines/v_express_pipeline.py:160). w fp32 [Cout, 9, C]. */
int vx_conv_out(const void* x, long long ldx, int NB, int H, int W, int C, int Cout, const float* w,
                const float* bias, void* out, long long sn, long long sc, int out_f32, int post, void* stream);

/* ---- tail of the tensor-core conv_out path: x [NB*HW, ldx] bf16 (conv3x3 output with Cout zero-padded to 32)
 * -> planar (n, co, y, x) with the optional image post-processing. */
int vx_extract_planar(const void* x, long long ldx, int NB, int HW, int Cout, void* out, long long sn, long long sc,
                      int out_f32, int post, void* stream);

/* ---- im2col of the stride-2 Downsample3D conv (modules/resnet.py:93-120) and nearest-2x upsample of
 * Upsample3D (:53-82), NHWC. */
int vx_im2col_s2(const void* x, int NB, int H, int W, int C, void* out, void* stream);
int vx_upsample2x(const void* x, int NB, int H, int W, int C, void* out, void* stream);

/* ---- time embedding: sinusoid (diffusers Timesteps, SURVEY.md B.4) and skinny linear (rows <= 8):
 * TimestepEmbedding (modules/unet_3d.py:464-470) and all 22 time_emb_proj at once (modules/resnet.py:225-228). */
int vx_timestep_embed(const float* t, int rows, int dim, float* out, void* stream);
int vx_skinny_linear(const float* x, int rows, int K, const void* w, const float* bias, int N, int act_in,
                     int act_out, float* y, void* stream);

/* ---- CFG combine + / num_frame_context + overlap accumulation for one window, and the DDIM v-prediction step
 * for all frames (pipelines/v_express_pipeline.py:548-572; diffusers DDIMScheduler.step, SURVEY.md B.5).
 * noise: ((b f),4,h,w) bf16; acc: fp32 (4, L, hw); latents: bf16 (4, L, hw) updated in place. */
int vx_cfg_overlap_accumulate(const void* noise, int f, int hw, int L, int do_cfg, const int* win, const int* count,
                              float guidance, float* acc, void* stream);
/* The same for n samples of one window in one launch (num_images_per_prompt): noise ((b n f),4,h,w) laid out
 * [uncond s0..s(n-1) | cond s0..s(n-1)] (b = 2) or [s0..s(n-1)] (b = 1), f frames per block; acc fp32 (n, 4, L, hw).
 * Per sample the rounding points and the skipped slots (win[i] = -1) are those of vx_cfg_overlap_accumulate, so sample s
 * accumulates the bits a one-sample call on its blocks would. */
int vx_cfg_overlap_accumulate_n(const void* noise, int n, int f, int hw, int L, int do_cfg, const int* win,
                                const int* count, float guidance, float* acc, void* stream);
/* vx_ddim_step is elementwise over n contiguous elements: for n samples pass latents / acc of shape (n, 4, L, hw) and
 * n * 4 * L * hw elements; every sample gets the update a one-sample call would give it. */
int vx_ddim_step(void* latents, const float* acc, long long n, float sqrt_a, float sqrt_1ma, float sqrt_aprev,
                 float sqrt_1maprev, void* stream);
/* Stochastic DDIM (eta > 0, diffusers DDIMScheduler.step with variance noise): vx_ddim_step with c_dir =
 * sqrt(1 - a_prev - sigma^2) in place of sqrt(1 - a_prev), then latents = bf16(prev + bf16(sigma * noise)).  noise is
 * fp32 with the layout of latents (n contiguous elements): the draw of the model dtype widened, so no rounding precedes
 * the multiply. */
int vx_ddim_step_eta(void* latents, const float* acc, const float* noise, long long n, float sqrt_a, float sqrt_1ma,
                     float sqrt_aprev, float c_dir, float sigma, void* stream);
/* vx_ddim_step on the k frames listed in `frames` (device int32, each in [0, L)) of latents bf16 / acc fp32, both
 * (ns, L, hw) with ns = samples x 4 channels, with the same rounding points; those acc entries are set to 0 in the same
 * pass.  Replaces the per-frame scheduler.step + noise_preds reset of the reference's streaming update
 * (pipelines/v_express_pipeline.py:566-572) for the wavefront order of VExpressPipeline.stream, where a frame is stepped
 * as soon as its last window has contributed and frames sit at different steps. */
int vx_ddim_step_frames(void* latents, float* acc, int ns, int L, int hw, const int* frames, int k, float sqrt_a,
                        float sqrt_1ma, float sqrt_aprev, float sqrt_1maprev, void* stream);
/* DPM-Solver++ multistep step (diffusers DPMSolverMultistepScheduler: dpmsolver++, midpoint, v-prediction) on n
 * contiguous elements of latents bf16, in place of the per-window scheduler.step of pipelines/v_express_pipeline.py:566-572.
 * With v = bf16(acc) and x the latent: m0 = bf16(bf16(alpha_s x) - bf16(sigma_s v)) (the x0 prediction);
 * order 1: latents = bf16(fp32(ratio x) - bf16(c0 m0));
 * order 2: D1 = bf16(inv_r0 bf16(m0 - x0_prev)), latents = bf16(fp32(ratio x) - bf16(c0 m0) - bf16(c0h D1)), in fp32
 * left to right.  x0_prev (bf16, the layout of latents) holds the previous step's m0 and receives this step's; order 1
 * does not read it.  Scalars from scheduler.dpm_coefficients. */
int vx_dpmpp_step(void* latents, const float* acc, void* x0_prev, long long n, float alpha_s, float sigma_s, float ratio,
                  float c0, float inv_r0, float c0h, int order, void* stream);
/* vx_dpmpp_step on the k frames listed in `frames` (device int32, each in [0, L)) of latents bf16 / acc fp32 / x0_prev
 * bf16, all (ns, L, hw), zeroing those acc entries in the same pass: the per-frame scheduler.step + noise_preds reset of
 * pipelines/v_express_pipeline.py:566-572 for the wavefront order of VExpressPipeline.stream (as vx_ddim_step_frames). */
int vx_dpmpp_step_frames(void* latents, float* acc, void* x0_prev, int ns, int L, int hw, const int* frames, int k,
                         float alpha_s, float sigma_s, float ratio, float c0, float inv_r0, float c0h, int order,
                         void* stream);

/* ---- post-processing of the decoded video (SURVEY.md 8f-f3): 3x3x3 median over (t, y, x) with reflect padding
 * (pipelines/utils.py:46-63) and the uint8 frames save_video hands to the encoder (:70-73, truncation of v*255).
 * video [C,T,H,W] fp32 (device); filtered (nullable) same layout; frames (nullable) [T,H,W,C] uint8.
 * Bit-exact vs the reference-generated golden (tests/test_zz_post_gpu.py). */
int vx_median3d_u8(const float* video, int C, int T, int H, int W, float* filtered, unsigned char* frames, void* stream);
/* The same filter on a run of frames, for a video decoded chunk by chunk (pipelines/utils.py:46-73 applied piecewise):
 * buf [C, nbuf, H, W] fp32 holds frames [buf_start, buf_start + nbuf) of a T-frame video and must include every temporal
 * neighbour of the owned frames [own_start, own_start + own_count) -- one halo frame on each side, time reflected only
 * at the video's true ends.  frames [own_count, H, W, C] uint8, bit-identical to those frames of vx_median3d_u8. */
int vx_median3d_range_u8(const float* buf, int C, int nbuf, int buf_start, int own_start, int own_count, int T, int H,
                         int W, unsigned char* frames, void* stream);

/* ---- nearest-2x upsample folded into the following 3x3 convolution (reference modules/resnet.py:53-90 Upsample3D;
 * diffusers Upsample2D in AutoencoderKL.decode): out = conv3x3(upsample2x(X)) computed as four 2x2 convolutions of X, one per
 * output parity class, with the 3x3 weights pre-summed per class (ops.pack_upconv_weight): Wt [4*Cout, 4*C]; out is the
 * NHWC [NB*2H*2W, ldc] upsampled image.  4/9 of the FLOPs, no 4x intermediate. */
int vx_upconv3x3_bf16(const void* X, int NB, int H, int W, int C, const void* Wt, int Cout, const float* bias, void* out,
                      long long ldc, int block_n, void* stream);

/* ---- 3x3 convolution with stride 2 on the tensor cores without a gathered copy of the input: the implicit-GEMM A boxes
 * are fetched through a TMA tensor map with traversal stride 2 along x and y.  X [NB,H,W,C] (H, W even), W [Cout, 9*C],
 * out [NB*(H/2)*(W/2), ldc].  pad_lo = 1: nn.Conv2d(stride=2, padding=1), the Downsample3D / Downsample2D of the denoising
 * UNet and the ReferenceNet (reference modules/resnet.py:93-120, modules/unet_3d_blocks.py:483-486, 620-623);
 * pad_lo = 0: F.pad(x, (0,1,0,1)) + padding 0, the Downsample2D(padding=0) of the VAE encoder (diffusers). */
int vx_conv3x3s2_bf16(const void* X, int NB, int H, int W, int C, const void* Wt, int Cout, const float* bias, int pad_lo,
                      void* out, long long ldc, int block_n, void* stream);

/* ---- conditioning prologue (SURVEY.md 8f-f2): im2col of a 3x3 conv (stride 1 or 2, pad 1, NHWC bf16) with an
 * optional SiLU on the gathered input; VKpsGuider's narrow conv -> SiLU chain (modules/v_kps_guider.py:35-45) runs as
 * im2col(SiLU(x)) + vx_gemm_bf16.  out [NB*Ho*Wo, 9*C], K order (tap, channel).  pad_lo = 1: pad 1 all round;
 * pad_lo = 0 (stride 2 only): pad (0,1,0,1), the Downsample2D(padding=0) of the VAE encoder (SURVEY.md 8f-f4). */
int vx_im2col3x3(const void* x, int NB, int H, int W, int C, int stride, int silu, int pad_lo, void* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VXH100_H */
