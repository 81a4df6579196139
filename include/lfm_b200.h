/* lfm_b200.h - C ABI of liblfm_b200.so: the H100-native latent flow-matching sampling path.
 *
 * Drop-in boundary for the sampling hot path of VinAIResearch/LFM.  The reference has no native code and
 * therefore no FFI of its own; each entry point below replaces a Python call site of the reference (cited as
 * reference-file:line) and is bound from Python with ctypes (see INTEGRATION.md for the stub a reference
 * maintainer would add).  Plain C: pointers, sizes, int status codes.  No torch types, no C++ exceptions.
 *
 * Conventions
 *  - All tensor pointers are DEVICE pointers on the ctx's device unless the name ends in _host.
 *  - Tensors use the reference's dtype and layout: latents/velocities fp32 NCHW contiguous [B, C, H, W];
 *    labels int64 [B]; times fp32.
 *  - The library BORROWS caller buffers for the duration of a call; it owns its weight copy and workspace.
 *  - Work is stream-ordered on `stream` (a cudaStream_t passed as void*; NULL = the legacy default stream).
 *  - Return value: 0 = ok, non-zero = error; lfm_last_error(ctx) (or lfm_last_error(NULL) for create
 *    failures) returns a message.  A ctx is bound to one device and is not thread-safe.
 */
#ifndef LFM_B200_H
#define LFM_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct lfm_ctx lfm_ctx;

enum { LFM_ARCH_DIT = 0, LFM_ARCH_UNET = 1 };
enum { LFM_DTYPE_F32 = 0 };
enum { LFM_METHOD_EULER = 0, LFM_METHOD_HEUN = 1, LFM_METHOD_MIDPOINT = 2, LFM_METHOD_RK4 = 3 };
/* bits of lfm_sample_fixed's `t_as_vector` argument */
enum { LFM_FIXED_T_VECTOR = 1, LFM_FIXED_PERTURB = 2 };
/* torchdiffeq's adaptive Runge-Kutta pairs (test_flow_latent.py:27 ADAPTIVE_SOLVER; dopri8 is not implemented) */
enum { LFM_ADAPTIVE_DOPRI5 = 0, LFM_ADAPTIVE_BOSH3 = 1, LFM_ADAPTIVE_HEUN = 2 };

/* Constructor arguments of the reference network (models/DiT.py:157-169, selected by
 * models/__init__.py:12-17 create_network).  image side = grid * patch. */
typedef struct lfm_model_desc {
    int32_t arch;            /* LFM_ARCH_DIT */
    int32_t img_resolution;  /* latent side, e.g. 32 */
    int32_t patch_size;      /* 2 */
    int32_t in_channels;     /* 4 */
    int32_t hidden_size;     /* D; multiple of 128; heads * 64 */
    int32_t depth;           /* L */
    int32_t num_heads;       /* H; head_dim must be 64 */
    int32_t mlp_hidden;      /* int(hidden_size * mlp_ratio) */
    int32_t table_rows;      /* y_embedder rows = num_classes + (label_dropout > 0) (models/DiT.py:79-81) */
} lfm_model_desc;

/* Constructor arguments of the reference ADM network (models/guided_diffusion/unet.py:407-428 as called by
 * get_flow_model, models/__init__.py:46-68).  Only the configuration the LFM presets use is implemented:
 * use_scale_shift_norm = True, resblock_updown = False, conv_resample = True, legacy attention order, dims = 2. */
typedef struct lfm_unet_desc {
    int32_t image_size;                /* latent side (config.image_size // 8), e.g. 64 */
    int32_t in_channels;               /* 4, or 5..16: concat-conditioned (see lfm_set_condition) */
    int32_t model_channels;            /* nf, multiple of 128 */
    int32_t out_channels;              /* 4 */
    int32_t num_res_blocks;
    int32_t n_attn_res;                /* number of entries used in attention_resolutions */
    int32_t attention_resolutions[8];  /* DOWNSAMPLE RATES at which attention is applied (unet.py:482) */
    int32_t n_mult;                    /* number of entries used in channel_mult */
    int32_t channel_mult[8];
    int32_t num_heads;
    int32_t num_head_channels;         /* -1: use num_heads */
    int32_t num_classes;               /* 0: unconditional; > 0: label_emb rows (y is then required) */
} lfm_unet_desc;

/* Constructor arguments of the reference EDM-style ADM network DhariwalUNet (models/EDM.py:716-735 as called by
 * get_edm_network, models/EDM.py:906-921, for `--model_type adm` without `--use_origin_adm`: the ffhq_adm / bed_adm /
 * imnet_adm presets).  channel_mult_emb = 4, channels_per_head = 64, augment_dim = 0, use_context = False. */
typedef struct lfm_edm_desc {
    int32_t img_resolution;       /* latent side (config.image_size // config.f), e.g. 32 */
    int32_t in_channels;          /* 4 */
    int32_t out_channels;         /* 4 */
    int32_t label_dim;            /* 0: unconditional; > 0: one-hot width of map_label */
    int32_t model_channels;       /* nf, multiple of 128 */
    int32_t n_mult;               /* number of entries used in channel_mult */
    int32_t channel_mult[8];
    int32_t num_blocks;           /* residual blocks per resolution (config.num_res_blocks) */
    int32_t n_attn_res;           /* number of entries used in attn_resolutions */
    int32_t attn_resolutions[8];  /* feature-map RESOLUTIONS with self-attention (EDM.py:788) */
} lfm_edm_desc;

/* Decoder half of the Stable-Diffusion AutoencoderKL the reference loads with
 * AutoencoderKL.from_pretrained(args.pretrained_autoencoder_ckpt) (test_flow_latent.py:131, test_flow_latent_ddp.py:57;
 * "stabilityai/sd-vae-ft-mse": block_out_channels (128, 256, 512, 512), layers_per_block 2, norm_num_groups 32,
 * latent_channels 4, out_channels 3).  diffusers is a third-party dependency outside /root/reference: the architecture
 * is restated in oracle/vae.py (parity unpinned). */
typedef struct lfm_vae_desc {
    int32_t latent_size;            /* latent side = image_size // 8: 16, 32 or 64 (128, 256, 512 pixel images) */
    int32_t latent_channels;        /* 4 */
    int32_t out_channels;           /* 3 */
    int32_t n_blocks;               /* number of entries used in block_out_channels */
    int32_t block_out_channels[8];  /* encoder order, e.g. 128, 256, 512, 512 (the decoder walks it backwards) */
    int32_t layers_per_block;       /* 2 => 3 ResnetBlock2D per decoder up-block */
    int32_t norm_num_groups;        /* 32 */
} lfm_vae_desc;

typedef struct lfm_ode_stats {
    int64_t nfe;       /* network evaluations */
    int64_t accepted;  /* dopri5 accepted steps */
    int64_t rejected;  /* dopri5 rejected steps */
} lfm_ode_stats;

/* models/__init__.py:6-17 create_network(config) -> nn.Module.  Creates an empty context on `device`. */
int lfm_create(const lfm_model_desc* desc, int device, lfm_ctx** out);

/* models/__init__.py:20-70 get_flow_model(config) -> UNetModel (config.use_origin_adm).  The same
 * lfm_set_param / lfm_finalize / lfm_forward / lfm_sample_* entry points then operate on the UNet
 * (model(t, x, y) = UNetModel.forward, unet.py:613-655; it has no forward_with_cfg: cfg_scale must be <= 1). */
int lfm_create_unet(const lfm_unet_desc* desc, int device, lfm_ctx** out);

/* Concat-conditioned UNetModel (in_channels in [5, 16], out_channels 4): the downstream tasks' WrapperCondFlow,
 * model(t, cat([x, cond], 1)) (downstream_tasks/test_flow_latent_inpainting.py, test_flow_latent_semantic_syn.py).
 * Copies cond [B_img, channels, H, W] fp32 NCHW (device), channels = in_channels - out_channels, into the context, ordered on
 * `stream`.  The samplers then evolve the [B_img, 4, H, W] state and evaluate the network on [state | cond]; they refuse to run
 * unless the stored condition holds exactly B_img images.  Their adaptive error norm covers the state only (torchdiffeq
 * integrates x; the concatenation happens inside the field).  The condition lives at a fixed address, so the cached step graphs
 * read each new condition.  lfm_forward on such a context takes x as the whole input [B, in_channels, H, W] and writes
 * v_out [B, 4, H, W]; it does not read the stored condition.  Refused on an unconditioned or unfinalized context, on a wrong
 * `channels` and on B_img above the finalized rows. */
int lfm_set_condition(lfm_ctx* ctx, const float* cond, int B_img, int channels, void* stream);

/* models/__init__.py:10-11 create_network(config) -> get_edm_network(config) -> DhariwalUNet (EDM.py:906-921).
 * The same lfm_set_param / lfm_finalize / lfm_forward / lfm_sample_* entry points then operate on it:
 * model(t, x, y) = DhariwalUNet.forward (EDM.py:812-845; y may be NULL even for a class-conditional net: the label
 * term is then skipped, :823) and cfg_scale > 1 = forward_with_cfg (EDM.py:847-861: the labels of the second half of
 * the batch are DROPPED - pass label_dim there, or anything: rows [B/2, B) of y are ignored).
 * State-dict keys as in the reference, including the constant `*.resample_filter` buffers of the up/down blocks
 * (accepted and checked to be 0.25). */
int lfm_create_edm(const lfm_edm_desc* desc, int device, lfm_ctx** out);

/* AutoencoderKL.from_pretrained(...) (test_flow_latent.py:131): a context for the DECODER.  lfm_set_param takes the
 * `decoder.*` and `post_quant_conv.*` entries of the diffusers state dict (attention projections under their current
 * names to_q / to_k / to_v / to_out.0); lfm_finalize(max_batch) sizes the workspace for max_batch images per call. */
int lfm_create_vae(const lfm_vae_desc* desc, int device, lfm_ctx** out);

/* first_stage_model.decode(z).sample (test_flow_latent.py:193, test_flow_latent_ddp.py:110; the caller divides the
 * latents by scale_factor as the reference does) and, optionally, the post-processing of the generation loop
 * (test_flow_latent_ddp.py:131-135) fused into the decoder's last kernel:
 *   z:       [B, 4, s, s] fp32 NCHW (device)
 *   out_f32: [B, 3, 8s, 8s] fp32 NCHW `sample`, or NULL
 *   out_u8:  [B, 8s, 8s, 3] uint8 = (clamp((sample + 1) / 2, 0, 1) * 255).permute(0, 2, 3, 1).to(uint8), or NULL */
int lfm_decode(lfm_ctx* ctx, const float* z, int B, float* out_f32, uint8_t* out_u8, void* stream);

/* AutoencoderKL(...).encode (downstream_tasks/test_flow_latent_inpainting.py:147): a context for the ENCODER, described by the
 * same struct, with out_channels read as the image channels (3) and latent_size = image side / 8 (16, 32 or 64).  lfm_set_param
 * takes the `encoder.*` and `quant_conv.*` entries of the diffusers state dict (attention projections under to_q / to_k / to_v /
 * to_out.0); a decoder key is refused, as an encoder key is by an lfm_create_vae context.  lfm_finalize(max_batch) sizes the
 * workspace for max_batch images per call. */
int lfm_create_vae_encoder(const lfm_vae_desc* desc, int device, lfm_ctx** out);

/* first_stage_model.encode(x).latent_dist's moments: quant_conv(encoder(x)).chunk(2) with the log-variance clamped to
 * [-30, 20], as DiagonalGaussianDistribution stores them.  The caller draws the sample (mean + exp(0.5 logvar) * eps).
 *   x:      [B, 3, S, S] fp32 NCHW (device), S = 8 latent_size
 *   mean:   [B, 4, S / 8, S / 8] fp32 NCHW
 *   logvar: [B, 4, S / 8, S / 8] fp32 NCHW
 * An lfm_create_vae context refuses this call; an lfm_create_vae_encoder context refuses lfm_decode. */
int lfm_encode(lfm_ctx* ctx, const float* x, int B, float* mean, float* logvar, void* stream);

/* The semantic-synthesis condition, cond_stage_model(one_hot(seg, num_cls).permute(0, 3, 1, 2).float())
 * (downstream_tasks/test_flow_latent_semantic_syn.py:94,131-135; models/encoder.py:90 SpatialRescaler with n_stages halvings,
 * method "bilinear", multiplier 0.5 and a bias-free 1x1 channel_mapper), computed from the labels without the one-hot:
 *   labels: [B, H, W] uint8 (device); H and W multiples of f = 2^n_stages, B * H * W < 2^31
 *   weight: [out_ch, num_classes] fp32 (channel_mapper.weight)
 *   out:    [B, out_ch, H / f, W / f] fp32 NCHW, out[b, k, i, j] = sum_c weight[k, c] * n_c / f^2 with n_c the count of class c
 *           in the label block [f i, f i + f) x [f j, f j + f), accumulated with one fmaf per class in class order.
 * 1 <= num_classes <= 256, 1 <= out_ch <= 16, 0 <= n_stages <= 4.  Labels >= num_classes are not counted (the caller validates
 * them).  No context: the work runs on the current device, stream-ordered on `stream`; errors through lfm_last_error(NULL). */
int lfm_label_condition(const uint8_t* labels, int B, int H, int W, int num_classes, int n_stages, const float* weight, int out_ch,
                        float* out, void* stream);

/* nn.Module.load_state_dict (test_flow_latent.py:142): one call per state-dict entry, `key` exactly as in the
 * reference state_dict (SURVEY.md 8(b)); `ptr` may be a host or a device pointer (fp32).  The data is copied
 * (GEMM weights are repacked to bf16; qkv and fc1 quantised to e4m3 in FP8 mode, see lfm_set_fp8).  Unknown key or wrong shape -> error (strict=True behaviour). */
int lfm_set_param(lfm_ctx* ctx, const char* key, const void* ptr, int dtype, const int64_t* shape, int ndim);

/* FP8 sampling mode of a DiT context (enable != 0; off by default), valid between lfm_create and lfm_set_param of the qkv
 * and fc1 weights.  Each block's attn.qkv and mlp.fc1 GEMMs then run on e4m3 operands (wgmma k32 e4m3, fp32 accumulation):
 * ln_modulate writes the LayerNorm + modulate output as e4m3 codes with one fp32 scale per token row (amax / 448), and the
 * two weights are quantised at upload, from the fp32 source after the qkv re-order and head padding, with one fp32 scale per
 * output channel; the context keeps only the e4m3 copies.  proj, fc2, attention and everything else stay as they are.  Not a
 * behaviour of the reference: its results differ from the bf16 path's by the e4m3 rounding of those operands.  Refused after
 * lfm_finalize, on UNet, EDM and VAE contexts, and once a qkv or fc1 weight has been uploaded in the other mode. */
int lfm_set_fp8(lfm_ctx* ctx, int enable);

/* After all parameters are set: checks that none is missing (strict), allocates the activation workspace for
 * up to `max_batch` network rows (2x images under CFG) and builds the TMA descriptors. */
int lfm_finalize(lfm_ctx* ctx, int max_batch);

/* model(t, x, y) / model.forward_with_cfg(t, x, y, cfg_scale)  (models/DiT.py:252-272, 274-290).
 *   t: [t_numel] fp32, t_numel == 1 (0-d t, broadcast) or B.   x, v_out: [B, C, H, W].   y: [B] int64 or NULL
 *   (NULL = the table's last row, models/DiT.py:259-260).
 *   cfg_scale <= 1: v_out = DiT(t, x, y).
 *   cfg_scale  > 1: forward_with_cfg - B must be even, rows [B/2, B) of y hold the null class; the first half
 *   of x is evaluated with both label halves and v_out = cat[g, g], g = u + s (c - u).
 *   Labels are validated by the caller (the Python mirror raises like nn.Embedding / one_hot would); on the device an
 *   out-of-range label is clamped to the table, never read out of bounds. */
int lfm_forward(lfm_ctx* ctx, const float* t, int t_numel, const float* x, const int64_t* y, int B, float cfg_scale,
                float* v_out, void* stream);

/* Fixed-step integration of dx/dt = v(t, x) over the nodes t_grid[0..n_grid) (device or host pointer, fp32):
 *   LFM_METHOD_EULER  x += v(t_i, x) (t_{i+1} - t_i)                sampler/karras_sample.py:86-118 and
 *                                                                   torchdiffeq fixed-grid euler (test_flow_latent.py:61-73)
 *   LFM_METHOD_HEUN   predictor + trapezoid corrector for intervals i < heun_corrector_limit, Euler beyond
 *                                                                   sampler/karras_sample.py:122-161
 *   LFM_METHOD_MIDPOINT / LFM_METHOD_RK4   torchdiffeq's fixed-grid midpoint and rk4 (3/8 rule) step functions
 *                                                                   (test_flow_latent.py:61-73 with --method midpoint|rk4)
 *   t_as_vector: bit 0 (LFM_FIXED_T_VECTOR): 0 = the model sees a 0-d t (torchdiffeq), 1 = a [B] vector (Karras samplers);
 *   bit 1 (LFM_FIXED_PERTURB): torchdiffeq options["perturb"] = True (test_flow_latent.py:44-48,64): the first evaluation of
 *   every step sees t one fp32 ulp past the node, rk4's last one one ulp before the next node.
 *   x_inout: [B_img, C, H, W] latents, updated in place.  y: labels, [B_img] (cfg_scale <= 1) or [2*B_img]
 *   (cfg_scale > 1: conditional labels then null labels; a 2*B_img-row network batch is evaluated per NFE).
 *   The whole trajectory runs from a captured CUDA graph; no host synchronisation between steps. */
int lfm_sample_fixed(lfm_ctx* ctx, int method, float* x_inout, const float* t_grid_host, int n_grid, int t_as_vector,
                     int heun_corrector_limit, const int64_t* y, int B_img, float cfg_scale, lfm_ode_stats* stats,
                     void* stream);

/* Adaptive Dormand-Prince 5(4) from t0 down to t1 with torchdiffeq's controller (rtol/atol, RMS norm over the
 * whole batch, fp64 time, dense output at t1)        test_flow_latent.py:42-76 with --method dopri5. */
int lfm_sample_dopri5(lfm_ctx* ctx, float* x_inout, double t0, double t1, double rtol, double atol, const int64_t* y,
                      int B_img, float cfg_scale, lfm_ode_stats* stats, void* stream);

/* The same controller with another embedded pair: --method dopri5 | bosh3 | adaptive_heun (test_flow_latent.py:27,61-73;
 * torchdiffeq rk_common.RKAdaptiveStepsizeODESolver: initial step with order - 1, step factor with order, y1 / f1 / dense
 * output as in its _runge_kutta_step / _interp_fit).  lfm_sample_dopri5 == lfm_sample_adaptive(LFM_ADAPTIVE_DOPRI5). */
int lfm_sample_adaptive(lfm_ctx* ctx, int method, float* x_inout, double t0, double t1, double rtol, double atol,
                        const int64_t* y, int B_img, float cfg_scale, lfm_ode_stats* stats, void* stream);

const char* lfm_last_error(const lfm_ctx* ctx);
void lfm_destroy(lfm_ctx* ctx);

/* Number of kernels the library has launched on this ctx since creation (bench.py's gpu_launches). */
int64_t lfm_launch_count(const lfm_ctx* ctx);

/* ---- kernel-level entry points used by the parity tests (tests/test_gpu_parity.py) ------------------- */
/* C = A[M,K] W[N,K]^T with epilogue `epi` (0 bias->bf16, 1 bias+gelu->bf16, 2 gated residual fp32, 3 bias->fp32).
 * a, w: bf16 device pointers.  block_n: tile width 128 or 256 (128 x block_n tiles), or 0 for the width the network would
 * pick for this shape; any other value is rejected. */
int lfm_dbg_gemm(const void* a_bf16, const void* w_bf16, const float* bias, void* out, const float* gate,
                 int gate_stride, int rows_per_sample, int M, int N, int K, int epi, int block_n, void* stream);
/* lfm_dbg_gemm with the persistent tile loop walking the 128-row blocks from the last to the first (the network sets this on
 * every other GEMM); same arguments and results. */
int lfm_dbg_gemm_reversed(const void* a_bf16, const void* w_bf16, const float* bias, void* out, const float* gate,
                          int gate_stride, int rows_per_sample, int M, int N, int K, int epi, int block_n, void* stream);
/* lfm_dbg_gemm with the epilogue's store path chosen by the caller, so that the paths can be compared in one build.  reverse:
 * as lfm_dbg_gemm_reversed when non-zero.  tma_store: -1 staged in shared memory and written by TMA stores whenever the output
 * allows it (16-byte aligned base and pitch; what lfm_dbg_gemm and the network do), 0 register stores, 1 TMA stores (rejected
 * when the output does not allow them).  Both paths write the same bits. */
int lfm_dbg_gemm_path(const void* a_bf16, const void* w_bf16, const float* bias, void* out, const float* gate,
                      int gate_stride, int rows_per_sample, int M, int N, int K, int epi, int block_n, int reverse,
                      int tma_store, void* stream);
/* The DiT's LayerNorm (no affine, eps 1e-6) + adaLN modulate: y[r] = bf16((x[r] - mean) rstd (1 + scale[b]) + shift[b]),
 * b = r / rows_per_sample, the vectors of sample b at shift / scale + b * mod_stride (0: one shared row).  x fp32 [M, D],
 * y bf16 [M, D].  D = 128 x {2, 3, 6, 8, 9}; rows_per_sample a multiple of 16; down 1 sweeps the rows downwards.  All pointers
 * 16-byte aligned, mod_stride a multiple of 4. */
int lfm_dbg_ln_modulate(const float* x, void* y_bf16, const float* shift, const float* scale, int mod_stride, int rows_per_sample,
                        int M, int D, int down, void* stream);
/* The FP8 mode's GEMM (lfm_set_fp8): out = bf16(epi(acc a_scale[m] w_scale[n] + bias[n])), acc = sum_k a[m, k] w[n, k] in fp32
 * over e4m3 codes a [M, K] and w [N, K] (device), a_scale fp32 [M], w_scale fp32 [N], bias fp32 [N] or NULL, out bf16 [M, N].
 * epi 0 (bias) or 1 (bias + GELU(tanh)); block_n 0 (the network's pick), 128 or 256.  K % 128 == 0, N % 8 == 0.  Arguments are
 * checked before the device is touched. */
int lfm_dbg_gemm_fp8(const void* a_e4m3, const float* a_scale, const void* w_e4m3, const float* w_scale, const float* bias,
                     void* out_bf16, int M, int N, int K, int epi, int block_n, void* stream);
/* lfm_dbg_ln_modulate with the FP8 mode's output: v = the modulated fp32 row, y_scale[r] = amax|v| / 448 (1 for an all-zero row),
 * y[r] = e4m3(v / y_scale[r]) (round to nearest even, saturating).  y e4m3 [M, D], y_scale fp32 [M]; other arguments as
 * lfm_dbg_ln_modulate. */
int lfm_dbg_ln_modulate_fp8(const float* x, void* y_e4m3, float* y_scale, const float* shift, const float* scale, int mod_stride,
                            int rows_per_sample, int M, int D, int down, void* stream);
/* The FP8 mode's weight quantiser: w fp32 [N, K] (device) -> scales fp32 [N] = amax|w[n, :]| / 448 (1 for an all-zero row) and
 * codes e4m3 [N, K] = e4m3(w / scales[n]) (round to nearest even, saturating). */
int lfm_dbg_quantize_rows_fp8(const float* w, void* codes_e4m3, float* scales, int N, int K, void* stream);
/* The conditioning stage of the DiT, ADM and EDM networks for `rows` rows, each step into a caller-allocated output: tf_out fp32
 * [rows, feat] timestep features [cos | sin] of t (t_numel 1 or rows), h1_out fp32 [rows, E] = SiLU(w0 tf + b0), c_bf16 bf16
 * [rows, E] = SiLU(w2 h1 + b2 + table[row]) with row = y ? clamp(y[r], 0, max_row) : null_row, and no table term when that is
 * -1.  The networks use max_row = null_row = table_rows - 1 (DiT), max_row = num_classes - 1 with null_row -1 (ADM), and
 * max_row = label_dim, the all-zero row after the labels, with null_row -1 (EDM).  w0 [E, feat], w2 [E, E], table [max_row + 1, E],
 * all fp32; feat and E multiples of 128 up to 4096.  table may be NULL when neither y nor null_row reads it. */
int lfm_dbg_condition(const float* t, int t_numel, const long long* y, int rows, int feat, int E, const float* w0, const float* b0,
                      const float* w2, const float* b2, const float* table, int max_row, int null_row, float* tf_out, float* h1_out,
                      void* c_bf16, void* stream);
/* The DiT's patch embed: M token rows of G x G tokens per sample, row m of sample b = m / G^2 reads latent b % x_rows of x (NCHW
 * fp32, C channels of side p G).  Wt fp32 [C p p, D] (the conv weight transposed, patch vector order (c, p, q)), bias [D],
 * pos [G^2, D] -> tok fp32 [M, D].  p 2 (C 4), 4 or 8; D a multiple of 4. */
int lfm_dbg_patch_embed(const float* x, int x_rows, const float* Wt, const float* bias, const float* pos, float* tok, int D, int G,
                        int C, int p, int M, void* stream);
/* The DiT's FinalLayer (LayerNorm, modulate with shift / scale + b * mod_stride, Linear(D, p p C)) and unpatchify: x fp32 [M, D]
 * -> v_net fp32 NCHW [M / G^2, C, p G, p G].  W fp32 [p p C, D] with out-feature (pp p + q) C + c, bias [p p C].  p 2 (C 4), 4 or
 * 8; D a multiple of 128 up to 1536; mod_stride a multiple of 4. */
int lfm_dbg_final_layer(const float* x, const float* shift, const float* scale, int mod_stride, const float* W, const float* bias,
                        float* v_net, int M, int D, int G, int C, int p, void* stream);
/* Layouts of the qkv rows of lfm_dbg_attention (row = the 3 heads ch features of one token):
 *   LFM_QKV_TIMM        {q,k,v} * heads ch + head * ch + c   (timm's Attention, the DiT checkpoints)
 *   LFM_QKV_HEAD_MAJOR  head * 3 ch + {q,k,v} * ch + c       (guided-diffusion's QKVAttentionLegacy) */
enum { LFM_QKV_TIMM = 0, LFM_QKV_HEAD_MAJOR = 1 };
/* One attention as the DiT and UNet programs run it, on the kernel and scale their route table picks for (T, ch, layout):
 * qkv bf16 [B*T, 3 heads ch] -> out bf16 [B*T, heads ch], softmax(q k^T / sqrt(head_dim)) v per (image, head).
 * ch is the stored head width; head_dim < ch means heads zero-padded from head_dim to ch channels (DiT-XL: 72 stored as 80),
 * which only the mma.sync kernels take.  Routes: timm layout: 256 tokens with ch 64 (TMA + wgmma).  Head-major: 16 / 64 tokens
 * with ch 64, 80, 128 or 256; other multiples of 64 tokens with ch 64 or 80; up to 256 tokens with ch a multiple of 8 up to 256
 * (SIMT, head_dim = ch).  Other shapes, a bad layout or head_dim, and B or heads < 1 are refused before the device is touched. */
int lfm_dbg_attention(const void* qkv_bf16, void* out_bf16, int B, int T, int heads, int ch, int head_dim, int layout, void* stream);
/* The UNet programs' 3x3 convolution (pad 1) as the implicit GEMM the network runs, built and launched by the network's own code.
 *   x: bf16 NHWC [B, side, side, Cin] (Cin % 64 == 0); stride 1 or 2 (output side side / stride: 4, 8, ..., 256).
 *   w: bf16 [Cout, 9 Cin], K index (r * 3 + s) * Cin + c (lfm_set_param's repacked order); bias: fp32 [Cout]; Cout 4 or % 8 == 0.
 *   out: [B, side/stride, side/stride, Cout]: epi 3 fp32 = conv + bias, 0 bf16 = conv + bias, 2 fp32 out += conv + bias.
 *   block_n: 0 = the network's tile width for the shape, or 128 / 256.
 *   ksplit: -1 = the network's split-K decision for B images, 1 = none, 2..8 = that many K slices (epi 3 / 2, block_n 0 / 128).
 *   gn_bins: NULL, or the GroupNorm statistics of the output taken in the epilogue (u64 [B][16 replicas][32 groups][sum, sum of
 *   squares], the sum in units of 2^-28 and the sum of squares in 2^-20; accumulated: the caller zeroes it).  Needs epi 3 / 0, no
 *   split-K, Cout / 32 in {4, 8, 16, 32, 64} and a multiple of 32 output pixels.
 * The entry allocates its own split-K scratch on `stream`. */
int lfm_dbg_conv(const void* x_bf16, const void* w_bf16, const float* bias, void* out, unsigned long long* gn_bins, int B, int side,
                 int Cin, int Cout, int stride, int block_n, int epi, int ksplit, void* stream);
/* The same convolution for output rows wider than one 128-pixel tile (the VAE decoder's 256- and 512-pixel stages, run on
 * 128-pixel row segments): side 256 or 512, stride 1, ksplit 1 (never split along K); x, w, bias, out, gn_bins, block_n and epi as
 * lfm_dbg_conv.  Arguments are checked before the device is touched. */
int lfm_dbg_conv_wide(const void* x_bf16, const void* w_bf16, const float* bias, void* out, unsigned long long* gn_bins, int B, int side,
                      int Cin, int Cout, int stride, int block_n, int epi, int ksplit, void* stream);
/* The VAE encoder's Downsample2D(padding=0), F.pad(x, (0, 1, 0, 1)) then a 3x3 stride-2 convolution, as the network runs it: the
 * extra bottom row and right column are the tensor map's zero fill.  side 8..512 (a power of 2; output rows wider than 128 pixels
 * run on 128-pixel row segments), stride 2; every other argument as lfm_dbg_conv.  Arguments are checked before the device is
 * touched. */
int lfm_dbg_conv_down(const void* x_bf16, const void* w_bf16, const float* bias, void* out, unsigned long long* gn_bins, int B, int side,
                      int Cin, int Cout, int stride, int block_n, int epi, int ksplit, void* stream);
/* The UNet programs' conv_in (3x3, pad 1, fp32) as the network runs it: input channels [a | b] of two NCHW fp32 sources, a with a_ch
 * channels and image i at a + i * a_stride, b likewise (NULL when b_ch = 0); a_ch + b_ch in [3, 16].  w fp32 [Cout, a_ch + b_ch, 3, 3],
 * bias fp32 [Cout], out fp32 NHWC [B, side, side, Cout].  side in [1, 256], or 512 with 3 channels (the VAE encoder's image input),
 * with (a_ch + b_ch) * 3 * (side + 4) floats in 48 KB.
 * Arguments are checked before the device is touched. */
int lfm_dbg_conv_in(const float* a, int a_ch, long long a_stride, const float* b, int b_ch, long long b_stride, const float* w,
                    const float* bias, float* out, int B, int side, int Cout, void* stream);
/* The VAE encoder's tail as lfm_encode runs it: in = conv_out's output, NHWC fp32 [B * HW, 8] (16-byte aligned); w fp32 [8, 8]
 * (quant_conv.weight), bias fp32 [8]; mean = quant_conv channels 0..3 and logvar = clamp(channels 4..7, -30, 20), NCHW fp32
 * [B, 4, HW].  Arguments are checked before the device is touched. */
int lfm_dbg_vae_quant(const float* in, const float* w, const float* bias, float* mean, float* logvar, int B, int HW, void* stream);
/* The batched GEMM of the VAE mid-block attention: M = B * out_hw rows in groups of batch_m; group g computes
 * out[g rows] = A[rows] W[g * b_batch_rows .. + N]^T (+ bias), A row = row % a_mod when a_mod > 0 (A shared by all groups).
 * a: bf16 [a_rows, K] with row pitch a_ld, w: bf16 [w_rows, K] with row pitch w_ld (column windows of wider matrices);
 * out [M, N] fp32 (epi 3) or bf16 (epi 0); bias fp32 [N] or NULL.  K % 64 == 0, N % 256 == 0, batch_m % 128 == 0. */
int lfm_dbg_gemm_batched(const void* a_bf16, int a_rows, int a_ld, const void* w_bf16, int w_rows, int w_ld, int K, int N, void* out,
                         const float* bias, int B, int out_hw, int epi, int batch_m, int a_mod, int b_batch_rows, void* stream);
/* The UNet programs' GroupNorm(32 groups) pass over B images of HW pixels, with the network's launch code.
 *   source: the channel concatenation [a (Ca channels) | b (Cb channels)] of fp32 NHWC tensors (b NULL when Cb = 0), C = Ca + Cb
 *   a multiple of 128 up to 2048; src_bf16: NULL, or the same values as bf16 [B, HW, C] to read instead.
 *   bins: NULL = the statistics pass over the fp32 source, in at most max_chunks pixel chunks per image (32 in the UNets, 256 in
 *   the VAE); else the statistics as lfm_dbg_conv's gn_bins.
 *   out = act(((x - mean) * rstd * gamma + beta) * (1 + film[c]) + film[C + c]): gamma, beta fp32 [C]; film NULL or fp32 rows
 *   [scale (C) | shift (C)] at film + b * film_stride; act 1 = SiLU; eps > 0.
 *   out bf16 [B, HW, C]; copy_out: NULL or fp32 [B, HW, C] = the source; raw_out: NULL or bf16 [B, HW, C] = the source as bf16. */
int lfm_dbg_groupnorm(const float* a, int Ca, const float* b, int Cb, const void* src_bf16, const unsigned long long* bins,
                      int max_chunks, const float* gamma, const float* beta, const float* film, int film_stride, int act, float eps,
                      void* out_bf16, float* copy_out, void* raw_out, int B, int HW, void* stream);
/* Intermediate activations of the last lfm_forward (fp32 token stream [B*T, D] after all blocks). */
int lfm_dbg_tokens(lfm_ctx* ctx, float* out, int B);

#ifdef __cplusplus
}
#endif
#endif /* LFM_B200_H */
