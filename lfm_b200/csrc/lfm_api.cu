// lfm_b200 - C ABI (include/lfm_b200.h): context, parameter upload, DiT forward, ODE solvers.
// Single translation unit; build:  nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -shared ...
#include "../../include/lfm_b200.h"

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <map>
#include <string>
#include <unordered_map>
#include <vector>

#include "common.cuh"
#include "gemm.cuh"
#include "attention_wgmma.cuh"
#include "kernels.cuh"
#include "unet.cuh"
#include "attention_flash.cuh"
#include "vae.cuh"

using namespace lfm;

// ------------------------------------------------------------------------------------------------
// errors

static thread_local std::string g_last_error;

struct lfm_ctx;
static int fail(lfm_ctx* ctx, const char* fmt, ...);

#define CUDA_OK(call)                                                                              \
    do {                                                                                           \
        cudaError_t _e = (call);                                                                   \
        if (_e != cudaSuccess)                                                                     \
            return fail(ctx, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(_e), __FILE__, __LINE__); \
    } while (0)

// ------------------------------------------------------------------------------------------------
// TMA descriptor encoding through the driver entry point (no -lcuda link dependency)

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (fn == nullptr) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}

// Row-major bf16 matrix [rows, cols]; box = 64 columns (one 128-byte swizzle row) x box_rows rows.
static bool make_tmap_bf16(CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols, uint32_t box_rows) {
    EncodeTiledFn fn = get_encode_fn();
    if (fn == nullptr) return false;
    cuuint64_t dims[2] = {cols, rows};
    cuuint64_t strides[1] = {cols * 2};
    cuuint32_t box[2] = {64, box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS;
}

static int env_int(const char* name, int dflt) {
    const char* v = getenv(name);
    return (v != nullptr && *v != 0) ? atoi(v) : dflt;
}

// ------------------------------------------------------------------------------------------------
// kernel launch helpers

// SM count of the device the calling thread is working on: set at every API entry from the ctx (a ctx is bound to
// one device; several contexts on different devices may live in one process).
static thread_local int g_num_sms = 0;

// Opt-in for more than 48 KB of dynamic shared memory.  cudaFuncSetAttribute applies to the CURRENT device only, so
// the "done" flag is kept per device (one bit each); safe to call from several host threads.
struct DevOnce {
    std::atomic<uint64_t> mask{0};
};
template <typename K>
static cudaError_t smem_opt_in(DevOnce& once, K kern, int bytes) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    const uint64_t bit = 1ull << (dev & 63);
    if (once.mask.load(std::memory_order_acquire) & bit) return cudaSuccess;
    e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e == cudaSuccess) once.mask.fetch_or(bit, std::memory_order_release);
    return e;
}
static int query_num_sms() {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 0;
    return n;
}

// Launch with (by default; LFM_PDL=0 disables) the programmatic-stream-serialization attribute: see pdl_wait() in common.cuh.
static int g_pdl = -1;
template <typename... KArgs, typename... Args>
static cudaError_t launch_k(void (*kern)(KArgs...), dim3 grid, unsigned block, size_t smem, cudaStream_t s, Args&&... args) {
    if (g_pdl < 0) g_pdl = env_int("LFM_PDL", 1);
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid;
    cfg.blockDim = dim3(block);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = s;
    cudaLaunchAttribute at[1];
    if (g_pdl) {
        at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        at[0].val.programmaticStreamSerializationAllowed = 1;
        cfg.attrs = at;
        cfg.numAttrs = 1;
    }
    return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}
// ONLY for kernels that execute pdl_wait() before their first global-memory access.

template <int BN, int EPI>
static cudaError_t launch_gemm_inst(cudaStream_t s, const CUtensorMap& ta, const CUtensorMap& tb, int M, int N, int K,
                                    const GemmEpi& ep, const ConvGeom& cg, int ksplit, int split_row_pitch) {
    static DevOnce once;
    auto kern = gemm_bf16_wgmma<BN, EPI>;
    if (cudaError_t e = smem_opt_in(once, kern, GemmCfg<BN>::kSmemBytes)) return e;
    const int items = ((M + kGemmBlockM - 1) / kGemmBlockM) * ((N + BN - 1) / BN) * ksplit;
    const int grid = items < g_num_sms ? items : g_num_sms;
    return launch_k(kern, dim3(grid), kGemmThreads, GemmCfg<BN>::kSmemBytes, s, ta, tb, M, N, K, ep, cg, ksplit, split_row_pitch);
}

// softmax(q k^T / 8) v for 256 tokens, head_dim 64, timm qkv order (attention_wgmma.cuh); tqkv: box {64, kGemmBoxRows} over [rows, 3 C]
static cudaError_t launch_attention_wgmma(cudaStream_t s, const CUtensorMap& tqkv, __nv_bfloat16* out, int C, int heads, int samples) {
    static DevOnce once;
    if (cudaError_t e = smem_opt_in(once, attention_wgmma_t256_d64, kAttnSmemBytes)) return e;
    const int items = samples * heads * 2;
    const int grid = items < g_num_sms ? items : g_num_sms;
    return launch_k(attention_wgmma_t256_d64, dim3(grid), kAttnThreads, kAttnSmemBytes, s, tqkv, out, C, heads, items,
                    0.125f * 1.4426950408889634f);
}

// Tile width: 256 columns, unless N fits in 128 or the 256-wide tiles would leave more than half of the SMs idle (small
// sampling batches) - then 128, which doubles the tiles of the launch.
static int pick_block_n(int M, int N) {
    const int tiles256 = ((M + kGemmBlockM - 1) / kGemmBlockM) * ((N + 255) / 256);
    return (N <= 128 || 2 * tiles256 <= g_num_sms) ? 128 : 256;
}

// A and W are tensor maps with a box of {64, kGemmBoxRows} (make_tmap_bf16 / make_tmap_act4d); block_n = 128 or 256
// (0: pick_block_n).  The batched GEMMs of ConvGeom need block_n 256 when N is a multiple of 256 (W rows of one group).
static cudaError_t launch_gemm(cudaStream_t s, const CUtensorMap& ta, const CUtensorMap& tb, int M, int N, int K, int epi,
                               int block_n, const GemmEpi& ep, const ConvGeom& cg = ConvGeom{0, 0, 0, 0, 1}, int ksplit = 1,
                               int split_row_pitch = 0) {
    if (block_n == 0) block_n = cg.batch_m > 0 ? 256 : pick_block_n(M, N);
#define LFM_GEMM_CASE(BN, E) \
    if (block_n == BN && epi == E) return launch_gemm_inst<BN, E>(s, ta, tb, M, N, K, ep, cg, ksplit, split_row_pitch);
    LFM_GEMM_CASE(256, EPI_BIAS_BF16)
    LFM_GEMM_CASE(256, EPI_BIAS_GELU_BF16)
    LFM_GEMM_CASE(256, EPI_GATE_RESID_F32)
    LFM_GEMM_CASE(256, EPI_BIAS_F32)
    LFM_GEMM_CASE(128, EPI_BIAS_BF16)
    LFM_GEMM_CASE(128, EPI_BIAS_GELU_BF16)
    LFM_GEMM_CASE(128, EPI_GATE_RESID_F32)
    LFM_GEMM_CASE(128, EPI_BIAS_F32)
#undef LFM_GEMM_CASE
    return cudaErrorInvalidValue;
}

template <int NV, int ROWS>
static cudaError_t launch_ln_inst2(cudaStream_t s, const float* x, __nv_bfloat16* y, const float* shift, const float* scale,
                                   int mod_stride, int rows_per_sample, int M, int order) {
    static DevOnce once;
    const int smem = ln_stages(NV, ROWS) * (ROWS + (ROWS == 16 ? 2 : 0)) * NV * 128 * 4;
    auto kern = ln_modulate_kernel<NV, ROWS>;
    if (cudaError_t e = smem_opt_in(once, kern, smem)) return e;
    const int tiles = (M + ROWS - 1) / ROWS;
    const int grid = tiles < g_num_sms ? tiles : g_num_sms;
    return launch_k(kern, dim3(grid), ROWS * 32, smem, s, x, y, shift, scale, mod_stride, rows_per_sample, M, order);
}
template <int NV>
static cudaError_t launch_ln_inst(cudaStream_t s, const float* x, __nv_bfloat16* y, const float* shift, const float* scale,
                                  int mod_stride, int rows_per_sample, int M, int order) {
    static const int rows = env_int("LFM_LN_ROWS", 16);  // 16-row ring by default; 8 / 0 / 32: the other shapes (A/B runs)
    if (rows == 16) return launch_ln_inst2<NV, 16>(s, x, y, shift, scale, mod_stride, rows_per_sample, M, order);
    if (rows == 0) {
        const int blocks = std::min((M + 7) / 8, 4 * g_num_sms);
        return launch_k(ln_modulate_direct_kernel<NV>, dim3(blocks), 256, 0, s, x, y, shift, scale, mod_stride, rows_per_sample, M, order);
    }
    if (rows == 32) {  // one persistent 32-warp block per SM, rows straight from global memory
        const int blocks = std::min((M + 31) / 32, g_num_sms);
        return launch_k(ln_modulate_direct_kernel<NV, 1024, 1>, dim3(blocks), 1024, 0, s, x, y, shift, scale, mod_stride, rows_per_sample, M, order);
    }
    return launch_ln_inst2<NV, 8>(s, x, y, shift, scale, mod_stride, rows_per_sample, M, order);
}
static cudaError_t launch_ln(cudaStream_t s, const float* x, __nv_bfloat16* y, const float* shift, const float* scale,
                             int mod_stride, int rows_per_sample, int M, int D, int order = 0) {
    switch (D / 128) {
        case 2: return launch_ln_inst<2>(s, x, y, shift, scale, mod_stride, rows_per_sample, M, order);
        case 3: return launch_ln_inst<3>(s, x, y, shift, scale, mod_stride, rows_per_sample, M, order);
        case 6: return launch_ln_inst<6>(s, x, y, shift, scale, mod_stride, rows_per_sample, M, order);
        case 8: return launch_ln_inst<8>(s, x, y, shift, scale, mod_stride, rows_per_sample, M, order);
        case 9: return launch_ln_inst<9>(s, x, y, shift, scale, mod_stride, rows_per_sample, M, order);
        default: return cudaErrorInvalidValue;
    }
}

static inline unsigned blocks_for(size_t n, int threads = 256) { return static_cast<unsigned>((n + threads - 1) / threads); }

// ------------------------------------------------------------------------------------------------
// context

struct ParamSlot {
    void* dst = nullptr;        // device destination (fp32 or bf16)
    std::vector<int64_t> shape;
    size_t numel = 0;
    bool to_bf16 = false;
    int kind = 0;  // 0 copy fp32, 1 cast bf16, 2 conv [Co,Ci,kh,kw] -> bf16 [Co,kh,kw,Ci], 3 out-conv -> fp32 [4][9][C],
                   // 4 fp32 transpose [R, rest] -> [rest, R], 5 / 6 EDM qkv weight / bias row re-order (aux0 = head dim,
                   // aux1 = target layout), 7 constant resample_filter (validated, not stored), 8 / 9 DiT qkv weight / bias rows
                   // re-ordered head-major for the mma.sync attention kernels (aux0 = head dim, aux1 = its stored, zero-padded width),
                   // 10 DiT proj weight with zero columns for the padded head channels
    int aux0 = 0, aux1 = 0;
    bool set = false;
};

struct BlockW {
    __nv_bfloat16 *w_qkv, *w_proj, *w_fc1, *w_fc2;
    float *b_qkv, *b_proj, *b_fc1, *b_fc2;
    CUtensorMap tm_qkv, tm_proj, tm_fc1, tm_fc2;
};

struct UNetState;

struct lfm_ctx {
    lfm_model_desc d{};
    int arch = LFM_ARCH_DIT;
    UNetState* un = nullptr;
    int device = 0;
    int num_sms = 0;
    int D = 0, L = 0, H = 0, T = 0, G = 0, C = 0, Hd = 0, Nmod = 0, HW = 0, chw = 0;
    int dh = 64, dhp = 64, Dq = 0;  // head_dim, its stored (zero-padded) width and the width H * dhp of the attention tensors
    bool qkv_head_major = false;    // qkv rows re-ordered head-major (everything but T = 256 with head_dim 64, see lfm_create)
    int max_rows = 0;
    bool finalized = false;
    std::string err;
    int64_t launches = 0;
    int zigzag = 0;        // LFM_ZIGZAG: alternate the row-sweep direction of consecutive kernels (L2 reuse)
    int l2_hint = 0;       // LFM_L2_HINT: evict_last L2 policy on the LayerNorm pass's loads of the residual stream

    std::unordered_map<std::string, ParamSlot> params;
    std::vector<void*> allocs;
    float* staging = nullptr;
    size_t staging_elems = 0;

    // parameters
    float *pos = nullptr, *pe_w = nullptr, *pe_b = nullptr, *t_w0 = nullptr, *t_b0 = nullptr, *t_w2 = nullptr,
          *t_b2 = nullptr, *ytable = nullptr, *fin_w = nullptr, *fin_b = nullptr, *b_mod = nullptr;
    __nv_bfloat16* w_mod = nullptr;
    CUtensorMap tm_wmod;
    std::vector<BlockW> blk;

    // workspace
    float *x_tok = nullptr, *mod = nullptr, *tfreq = nullptr, *h1 = nullptr, *v_net = nullptr;
    __nv_bfloat16 *xn = nullptr, *qkv = nullptr, *attn = nullptr, *hmid = nullptr, *c_silu = nullptr;
    CUtensorMap tm_xn, tm_attn, tm_hmid, tm_csilu;
    CUtensorMap tm_qkv_attn;  // qkv as read by the 256-token attention (timm order only)

    // solver state
    cudaStream_t stream = nullptr;
    cudaEvent_t ev_in = nullptr, ev_out = nullptr;
    float *x_state = nullptr, *x_pred = nullptr, *v_eff = nullptr, *d_prime = nullptr, *t_grid = nullptr,
          *t_eval = nullptr, *coef = nullptr, *ratio = nullptr, *y_stage = nullptr;
    float* kbuf[7] = {nullptr};
    double* partial = nullptr;
    long long* y_buf = nullptr;
    StepState* step_state = nullptr;
    float* ratio_host = nullptr;  // pinned
    DpStep* dp_dev = nullptr;     // dopri5: parameters of the step being attempted (device copy read by the step graph)
    DpStep* dp_host = nullptr;    // pinned
    struct StepGraph {
        cudaGraphExec_t exec = nullptr;
        int launches = 0;  // kernels per replay (measured on the warm-up run)
    };
    std::map<std::string, StepGraph> graphs;
};

static int fail(lfm_ctx* ctx, const char* fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_last_error = buf;
    if (ctx != nullptr) ctx->err = buf;
    return 1;
}

template <typename Tp>
static int dev_alloc(lfm_ctx* ctx, Tp** p, size_t count) {
    void* q = nullptr;
    CUDA_OK(cudaMalloc(&q, count * sizeof(Tp) + 256));
    CUDA_OK(cudaMemset(q, 0, count * sizeof(Tp) + 256));
    ctx->allocs.push_back(q);
    *p = static_cast<Tp*>(q);
    return 0;
}

static void add_param(lfm_ctx* ctx, const std::string& key, void* dst, std::vector<int64_t> shape, bool to_bf16) {
    ParamSlot s;
    s.dst = dst;
    s.shape = shape;
    s.numel = 1;
    for (int64_t v : shape) s.numel *= static_cast<size_t>(v);
    s.to_bf16 = to_bf16;
    s.kind = to_bf16 ? 1 : 0;
    ctx->params[key] = s;
}
static void add_param_kind(lfm_ctx* ctx, const std::string& key, void* dst, std::vector<int64_t> shape, int kind) {
    add_param(ctx, key, dst, shape, kind != 0);
    ctx->params[key].kind = kind;
}

static void add_param_aux(lfm_ctx* ctx, const std::string& key, void* dst, std::vector<int64_t> shape, int kind, int aux0, int aux1) {
    add_param_kind(ctx, key, dst, shape, kind);
    ctx->params[key].aux0 = aux0;
    ctx->params[key].aux1 = aux1;
}

extern "C" int lfm_create(const lfm_model_desc* desc, int device, lfm_ctx** out) {
    lfm_ctx* ctx = nullptr;
    if (desc == nullptr || out == nullptr) return fail(nullptr, "lfm_create: null argument");
    if (desc->arch != LFM_ARCH_DIT) return fail(nullptr, "lfm_create: unsupported arch %d", desc->arch);
    // Geometries (models/DiT.py:355-415; img_resolution = image_size // f): patch 2 / 4 / 8 on latents whose token grid is
    // 4 x 4, 8 x 8, 16 x 16 or 32 x 32 - e.g. /2 on 32 x 32 (every released preset) or 64 x 64, /4 on 64 x 64 or 32 x 32, /8 on 32 x 32.
    if (desc->patch_size != 2 && desc->patch_size != 4 && desc->patch_size != 8)
        return fail(nullptr, "lfm_create: patch_size must be 2, 4 or 8 (got %d)", desc->patch_size);
    {
        const int g = desc->img_resolution / desc->patch_size;
        if (desc->img_resolution <= 0 || desc->img_resolution % desc->patch_size != 0 || !(g == 4 || g == 8 || g == 16 || g == 32))
            return fail(nullptr, "lfm_create: the token grid (img_resolution / patch_size) must be 4, 8, 16 or 32 per side, i.e. 16, 64, "
                        "256 or 1024 tokens (got img_resolution %d, patch_size %d)", desc->img_resolution, desc->patch_size);
    }
    {
        const int nv = desc->hidden_size / 128;
        if (desc->hidden_size % 128 != 0 || !(nv == 2 || nv == 3 || nv == 6 || nv == 8 || nv == 9))
            return fail(nullptr, "lfm_create: hidden_size must be one of 256, 384, 768, 1024, 1152 (got %d)", desc->hidden_size);
    }
    if (desc->num_heads <= 0 || (desc->num_heads * 64 != desc->hidden_size && desc->num_heads * 72 != desc->hidden_size))
        return fail(nullptr, "lfm_create: head_dim must be 64 or 72 (hidden %d, heads %d)", desc->hidden_size, desc->num_heads);
    if (desc->mlp_hidden % 64 != 0) return fail(nullptr, "lfm_create: mlp_hidden must be a multiple of 64");
    if (desc->in_channels != 4) return fail(nullptr, "lfm_create: in_channels must be 4");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
        return fail(nullptr, "lfm_create: no CUDA device (liblfm_b200 has no CPU path)");
    if (device < 0 || device >= ndev) return fail(nullptr, "lfm_create: bad device %d", device);
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return fail(nullptr, "cudaGetDeviceProperties failed");
    if (prop.major != 9) return fail(nullptr, "lfm_create: device %d is sm_%d%d; this library is sm_90a only", device, prop.major, prop.minor);
    ctx = new lfm_ctx();
    ctx->d = *desc;
    ctx->device = device;
    CUDA_OK(cudaSetDevice(device));
    g_num_sms = ctx->num_sms = prop.multiProcessorCount;
    ctx->D = desc->hidden_size;
    ctx->L = desc->depth;
    ctx->H = desc->num_heads;
    ctx->G = desc->img_resolution / desc->patch_size;
    ctx->T = ctx->G * ctx->G;
    ctx->C = desc->in_channels;
    ctx->Hd = desc->mlp_hidden;
    ctx->HW = desc->img_resolution;
    ctx->chw = ctx->C * ctx->HW * ctx->HW;
    ctx->Nmod = (6 * ctx->L + 2) * ctx->D;
    ctx->zigzag = env_int("LFM_ZIGZAG", 1);
    ctx->l2_hint = env_int("LFM_L2_HINT", 0);
    const int D = ctx->D, L = ctx->L, Hd = ctx->Hd, T = ctx->T;
    const int ps = desc->patch_size;
    const int P = ctx->C * ps * ps;  // elements of one patch = out-features of the final linear
    // 256 tokens with head_dim 64 (every released preset) keep the checkpoint's timm qkv order, which the flash kernel reads directly.
    // Everything else - 16 / 64 / 1024 tokens, head_dim 72 (DiT-XL, stored padded to 80) - stores the qkv rows head-major.
    ctx->dh = desc->hidden_size / desc->num_heads;
    ctx->dhp = ctx->dh == 72 ? 80 : 64;
    ctx->Dq = desc->num_heads * ctx->dhp;
    ctx->qkv_head_major = (T != 256 || ctx->dh != 64);
    const bool qkv_head_major = ctx->qkv_head_major;
    const int Dq = ctx->Dq;

    if (dev_alloc(ctx, &ctx->pos, (size_t)T * D)) return 1;
    if (dev_alloc(ctx, &ctx->pe_w, (size_t)D * P)) return 1;
    if (dev_alloc(ctx, &ctx->pe_b, D)) return 1;
    if (dev_alloc(ctx, &ctx->t_w0, (size_t)D * 256)) return 1;
    if (dev_alloc(ctx, &ctx->t_b0, D)) return 1;
    if (dev_alloc(ctx, &ctx->t_w2, (size_t)D * D)) return 1;
    if (dev_alloc(ctx, &ctx->t_b2, D)) return 1;
    if (dev_alloc(ctx, &ctx->ytable, (size_t)desc->table_rows * D)) return 1;
    if (dev_alloc(ctx, &ctx->fin_w, (size_t)P * D)) return 1;
    if (dev_alloc(ctx, &ctx->fin_b, P)) return 1;
    if (dev_alloc(ctx, &ctx->w_mod, (size_t)ctx->Nmod * D)) return 1;
    if (dev_alloc(ctx, &ctx->b_mod, ctx->Nmod)) return 1;
    add_param(ctx, "pos_embed", ctx->pos, {1, T, D}, false);
    add_param_kind(ctx, "x_embedder.proj.weight", ctx->pe_w, {D, 4, ps, ps}, 4);  // stored transposed [P, D]
    add_param(ctx, "x_embedder.proj.bias", ctx->pe_b, {D}, false);
    add_param(ctx, "t_embedder.mlp.0.weight", ctx->t_w0, {D, 256}, false);
    add_param(ctx, "t_embedder.mlp.0.bias", ctx->t_b0, {D}, false);
    add_param(ctx, "t_embedder.mlp.2.weight", ctx->t_w2, {D, D}, false);
    add_param(ctx, "t_embedder.mlp.2.bias", ctx->t_b2, {D}, false);
    add_param(ctx, "y_embedder.embedding_table.weight", ctx->ytable, {desc->table_rows, D}, false);
    add_param(ctx, "final_layer.linear.weight", ctx->fin_w, {P, D}, false);
    add_param(ctx, "final_layer.linear.bias", ctx->fin_b, {P}, false);
    add_param(ctx, "final_layer.adaLN_modulation.1.weight", ctx->w_mod + (size_t)6 * L * D * D, {2 * D, D}, true);
    add_param(ctx, "final_layer.adaLN_modulation.1.bias", ctx->b_mod + (size_t)6 * L * D, {2 * D}, false);
    ctx->blk.resize(L);
    for (int i = 0; i < L; ++i) {
        BlockW& b = ctx->blk[i];
        if (dev_alloc(ctx, &b.w_qkv, (size_t)3 * Dq * D)) return 1;
        if (dev_alloc(ctx, &b.w_proj, (size_t)D * Dq)) return 1;
        if (dev_alloc(ctx, &b.w_fc1, (size_t)Hd * D)) return 1;
        if (dev_alloc(ctx, &b.w_fc2, (size_t)D * Hd)) return 1;
        if (dev_alloc(ctx, &b.b_qkv, 3 * Dq)) return 1;
        if (dev_alloc(ctx, &b.b_proj, D)) return 1;
        if (dev_alloc(ctx, &b.b_fc1, Hd)) return 1;
        if (dev_alloc(ctx, &b.b_fc2, D)) return 1;
        const std::string p = "blocks." + std::to_string(i) + ".";
        if (qkv_head_major) {
            add_param_aux(ctx, p + "attn.qkv.weight", b.w_qkv, {3 * D, D}, 8, ctx->dh, ctx->dhp);
            add_param_aux(ctx, p + "attn.qkv.bias", b.b_qkv, {3 * D}, 9, ctx->dh, ctx->dhp);
        } else {
            add_param(ctx, p + "attn.qkv.weight", b.w_qkv, {3 * D, D}, true);
            add_param(ctx, p + "attn.qkv.bias", b.b_qkv, {3 * D}, false);
        }
        if (ctx->dhp != ctx->dh)
            add_param_aux(ctx, p + "attn.proj.weight", b.w_proj, {D, D}, 10, ctx->dh, ctx->dhp);  // zero columns for the padded channels
        else
            add_param(ctx, p + "attn.proj.weight", b.w_proj, {D, D}, true);
        add_param(ctx, p + "attn.proj.bias", b.b_proj, {D}, false);
        add_param(ctx, p + "mlp.fc1.weight", b.w_fc1, {Hd, D}, true);
        add_param(ctx, p + "mlp.fc1.bias", b.b_fc1, {Hd}, false);
        add_param(ctx, p + "mlp.fc2.weight", b.w_fc2, {D, Hd}, true);
        add_param(ctx, p + "mlp.fc2.bias", b.b_fc2, {D}, false);
        add_param(ctx, p + "adaLN_modulation.1.weight", ctx->w_mod + (size_t)i * 6 * D * D, {6 * D, D}, true);
        add_param(ctx, p + "adaLN_modulation.1.bias", ctx->b_mod + (size_t)i * 6 * D, {6 * D}, false);
    }
    CUDA_OK(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
    CUDA_OK(cudaEventCreateWithFlags(&ctx->ev_in, cudaEventDisableTiming));
    CUDA_OK(cudaEventCreateWithFlags(&ctx->ev_out, cudaEventDisableTiming));
    *out = ctx;
    return 0;
}

extern "C" int lfm_set_param(lfm_ctx* ctx, const char* key, const void* ptr, int dtype, const int64_t* shape, int ndim) {
    if (ctx == nullptr || key == nullptr || ptr == nullptr) return fail(ctx, "lfm_set_param: null argument");
    if (dtype != LFM_DTYPE_F32) return fail(ctx, "lfm_set_param(%s): only fp32 sources are accepted", key);
    auto it = ctx->params.find(key);
    if (it == ctx->params.end()) return fail(ctx, "lfm_set_param: unexpected key '%s' (strict)", key);
    ParamSlot& s = it->second;
    if (ndim != (int)s.shape.size()) return fail(ctx, "lfm_set_param(%s): rank %d, expected %d", key, ndim, (int)s.shape.size());
    for (int i = 0; i < ndim; ++i)
        if (shape[i] != s.shape[i])
            return fail(ctx, "lfm_set_param(%s): dim %d is %lld, expected %lld", key, i, (long long)shape[i], (long long)s.shape[i]);
    CUDA_OK(cudaSetDevice(ctx->device));
    g_num_sms = ctx->num_sms;
    if (!s.to_bf16) {
        CUDA_OK(cudaMemcpy(s.dst, ptr, s.numel * sizeof(float), cudaMemcpyDefault));
    } else {
        if (ctx->staging_elems < s.numel) {
            if (ctx->staging != nullptr) CUDA_OK(cudaFree(ctx->staging));
            ctx->staging = nullptr;
            CUDA_OK(cudaMalloc(&ctx->staging, s.numel * sizeof(float)));
            ctx->staging_elems = s.numel;
        }
        CUDA_OK(cudaMemcpy(ctx->staging, ptr, s.numel * sizeof(float), cudaMemcpyDefault));
        if (s.kind == 2) {
            const int taps = static_cast<int>(s.shape[2] * s.shape[3]);
            conv_weight_repack_kernel<<<blocks_for(s.numel), 256>>>(ctx->staging, static_cast<__nv_bfloat16*>(s.dst),
                                                                   static_cast<int>(s.shape[0]), static_cast<int>(s.shape[1]), taps);
        } else if (s.kind == 4) {
            const int r0 = static_cast<int>(s.shape[0]);
            transpose_f32_kernel<<<blocks_for(s.numel), 256>>>(ctx->staging, static_cast<float*>(s.dst), r0,
                                                              static_cast<int>(s.numel / r0));
        } else if (s.kind == 3) {
            conv_out_weight_repack_kernel<<<blocks_for(s.numel), 256>>>(ctx->staging, static_cast<float*>(s.dst),
                                                                       static_cast<int>(s.shape[1]));
        } else if (s.kind == 5) {
            edm_qkv_weight_repack_kernel<<<blocks_for(s.numel), 256>>>(ctx->staging, static_cast<__nv_bfloat16*>(s.dst),
                                                                      static_cast<int>(s.shape[1]), s.aux0, s.aux1);
        } else if (s.kind == 6) {
            edm_qkv_bias_repack_kernel<<<blocks_for(s.numel), 256>>>(ctx->staging, static_cast<float*>(s.dst),
                                                                    static_cast<int>(s.shape[0] / 3), s.aux0, s.aux1);
        } else if (s.kind == 8) {  // aux0 = head_dim, aux1 = stored head width: the destination has 3 * heads * aux1 rows
            const int Dm = static_cast<int>(s.shape[1]);
            const size_t out_n = static_cast<size_t>(3) * (Dm / s.aux0) * s.aux1 * Dm;
            dit_qkv_weight_repack_kernel<<<blocks_for(out_n), 256>>>(ctx->staging, static_cast<__nv_bfloat16*>(s.dst), Dm, s.aux0, s.aux1);
        } else if (s.kind == 9) {
            const int Dm = static_cast<int>(s.shape[0] / 3);
            dit_qkv_bias_repack_kernel<<<blocks_for(static_cast<size_t>(3) * (Dm / s.aux0) * s.aux1), 256>>>(
                ctx->staging, static_cast<float*>(s.dst), Dm, s.aux0, s.aux1);
        } else if (s.kind == 10) {
            const int Dm = static_cast<int>(s.shape[0]);
            const size_t out_n = static_cast<size_t>(Dm) * (Dm / s.aux0) * s.aux1;
            dit_proj_weight_pad_kernel<<<blocks_for(out_n), 256>>>(ctx->staging, static_cast<__nv_bfloat16*>(s.dst), Dm, s.aux0, s.aux1);
        } else if (s.kind == 7) {
            float h[4] = {0.f, 0.f, 0.f, 0.f};
            CUDA_OK(cudaMemcpy(h, ctx->staging, sizeof(h), cudaMemcpyDeviceToHost));
            for (float v : h)
                if (v != 0.25f) return fail(ctx, "lfm_set_param(%s): resample_filter must be [[0.25, 0.25], [0.25, 0.25]] (EDM.py:96-98)", key);
        } else {
            f32_to_bf16_kernel<<<blocks_for((s.numel + 3) / 4), 256>>>(ctx->staging, static_cast<__nv_bfloat16*>(s.dst), s.numel);
        }
        CUDA_OK(cudaGetLastError());
        CUDA_OK(cudaDeviceSynchronize());
    }
    s.set = true;
    return 0;
}

static int alloc_solver_state(lfm_ctx* ctx, int R) {
    // solver state (sized for R latent rows)
    const size_t nst = (size_t)R * ctx->chw;
    if (dev_alloc(ctx, &ctx->x_state, nst)) return 1;
    if (dev_alloc(ctx, &ctx->x_pred, nst)) return 1;
    if (dev_alloc(ctx, &ctx->v_eff, nst)) return 1;
    if (dev_alloc(ctx, &ctx->d_prime, nst)) return 1;
    if (dev_alloc(ctx, &ctx->y_stage, nst)) return 1;
    for (int j = 0; j < 7; ++j)
        if (dev_alloc(ctx, &ctx->kbuf[j], nst)) return 1;
    if (dev_alloc(ctx, &ctx->t_grid, 8192 + 64)) return 1;
    if (dev_alloc(ctx, &ctx->t_eval, 8)) return 1;
    if (dev_alloc(ctx, &ctx->coef, 64)) return 1;
    if (dev_alloc(ctx, &ctx->ratio, 8)) return 1;
    if (dev_alloc(ctx, &ctx->partial, kRmsBlocks)) return 1;
    if (dev_alloc(ctx, &ctx->y_buf, (size_t)R)) return 1;
    if (dev_alloc(ctx, &ctx->step_state, 1)) return 1;
    CUDA_OK(cudaMallocHost(&ctx->ratio_host, 64));
    if (dev_alloc(ctx, &ctx->dp_dev, 1)) return 1;
    CUDA_OK(cudaMallocHost(&ctx->dp_host, sizeof(DpStep)));
    return 0;
}

static int unet_finalize(lfm_ctx* ctx, int R);

extern "C" int lfm_finalize(lfm_ctx* ctx, int max_batch) {
    if (ctx == nullptr) return fail(ctx, "lfm_finalize: null ctx");
    if (max_batch < 1) return fail(ctx, "lfm_finalize: max_batch must be >= 1");
    for (auto& kv : ctx->params)
        if (!kv.second.set) return fail(ctx, "lfm_finalize: missing key '%s' (strict)", kv.first.c_str());
    if (ctx->finalized && max_batch <= ctx->max_rows) return 0;
    if (ctx->finalized) return fail(ctx, "lfm_finalize: already finalized for %d rows; create a new ctx for %d", ctx->max_rows, max_batch);
    CUDA_OK(cudaSetDevice(ctx->device));
    g_num_sms = ctx->num_sms;
    if (ctx->arch == LFM_ARCH_UNET) {
        if (unet_finalize(ctx, max_batch)) return 1;
        if (alloc_solver_state(ctx, max_batch)) return 1;
        ctx->max_rows = max_batch;
        ctx->finalized = true;
        return 0;
    }
    const int D = ctx->D, Hd = ctx->Hd, T = ctx->T, R = max_batch, Dq = ctx->Dq;
    const size_t M = (size_t)R * T;
    const int Rpad = R < 128 ? 128 : R;
    if (dev_alloc(ctx, &ctx->x_tok, M * D)) return 1;
    if (dev_alloc(ctx, &ctx->xn, M * D)) return 1;
    if (dev_alloc(ctx, &ctx->qkv, M * 3 * Dq)) return 1;
    if (dev_alloc(ctx, &ctx->attn, M * Dq)) return 1;
    if (dev_alloc(ctx, &ctx->hmid, M * Hd)) return 1;
    if (dev_alloc(ctx, &ctx->mod, (size_t)R * ctx->Nmod)) return 1;
    if (dev_alloc(ctx, &ctx->c_silu, (size_t)Rpad * D)) return 1;
    if (dev_alloc(ctx, &ctx->tfreq, (size_t)R * 256)) return 1;
    if (dev_alloc(ctx, &ctx->h1, (size_t)R * D)) return 1;
    if (dev_alloc(ctx, &ctx->v_net, (size_t)R * ctx->chw)) return 1;
    if (alloc_solver_state(ctx, R)) return 1;

    bool ok = true;
    ok &= make_tmap_bf16(&ctx->tm_xn, ctx->xn, M, D, kGemmBoxRows);
    ok &= make_tmap_bf16(&ctx->tm_attn, ctx->attn, M, Dq, kGemmBoxRows);
    ok &= make_tmap_bf16(&ctx->tm_hmid, ctx->hmid, M, Hd, kGemmBoxRows);
    ok &= make_tmap_bf16(&ctx->tm_csilu, ctx->c_silu, Rpad, D, kGemmBoxRows);
    ok &= make_tmap_bf16(&ctx->tm_wmod, ctx->w_mod, ctx->Nmod, D, kGemmBoxRows);
    if (!ctx->qkv_head_major) ok &= make_tmap_bf16(&ctx->tm_qkv_attn, ctx->qkv, M, 3 * Dq, kGemmBoxRows);
    for (auto& b : ctx->blk) {
        ok &= make_tmap_bf16(&b.tm_qkv, b.w_qkv, 3 * Dq, D, kGemmBoxRows);
        ok &= make_tmap_bf16(&b.tm_proj, b.w_proj, D, Dq, kGemmBoxRows);
        ok &= make_tmap_bf16(&b.tm_fc1, b.w_fc1, Hd, D, kGemmBoxRows);
        ok &= make_tmap_bf16(&b.tm_fc2, b.w_fc2, D, Hd, kGemmBoxRows);
    }
    if (!ok) return fail(ctx, "lfm_finalize: cuTensorMapEncodeTiled failed");
    ctx->max_rows = R;
    ctx->finalized = true;
    return 0;
}

// ------------------------------------------------------------------------------------------------
// the velocity network: rows network rows, latents x has x_rows samples (row b reads sample b % x_rows)

#define LAUNCH_OK()                                   \
    do {                                              \
        CUDA_OK(cudaGetLastError());                  \
        ctx->launches++;                              \
    } while (0)
#define LAUNCH_K(...)                                 \
    do {                                              \
        CUDA_OK(launch_k(__VA_ARGS__));               \
        ctx->launches++;                              \
    } while (0)

static int check_ready(lfm_ctx* ctx, int rows, const char* who);

#include "unet_host.inc"
#include "vae_host.inc"

static int ctx_unet_variant(const lfm_ctx* ctx) { return ctx->un != nullptr ? ctx->un->variant : 0; }

static int launch_network(lfm_ctx* ctx, cudaStream_t s, const float* t, int t_numel, const float* x, int x_rows,
                          const long long* y, int rows) {
    if (ctx->arch == LFM_ARCH_UNET) return launch_unet(ctx, s, t, t_numel, x, x_rows, y, rows);
    const int D = ctx->D, L = ctx->L, Hd = ctx->Hd, T = ctx->T, Dq = ctx->Dq;
    const int M = rows * T;
    // Conditioning c = t_emb(t) + y_emb(y) and the adaLN tables.  A 0-d t with y = None (every unconditional
    // preset) gives the same c for every row: compute ONE row and let all samples read it (table stride 0).
    const bool uniform_c = (t_numel == 1 && y == nullptr);
    const int crows = uniform_c ? 1 : rows;
    const int Nmod = uniform_c ? 0 : ctx->Nmod;  // stride between samples in the modulation table
    timestep_features_kernel<<<crows, 256, 0, s>>>(t, t_numel, ctx->tfreq, crows);
    LAUNCH_OK();
    skinny_linear_kernel<0><<<(D + 7) / 8, 256, 0, s>>>(ctx->t_w0, ctx->t_b0, ctx->tfreq, crows, D, 256, nullptr, nullptr,
                                                        0, ctx->h1, nullptr);
    LAUNCH_OK();
    skinny_linear_kernel<1><<<(D + 7) / 8, 256, 0, s>>>(ctx->t_w2, ctx->t_b2, ctx->h1, crows, D, D, ctx->ytable, y,
                                                        ctx->d.table_rows - 1, nullptr, ctx->c_silu);
    LAUNCH_OK();
    {   // all adaLN modulation vectors of the network in one GEMM: mod[crows, (6L+2) D]
        GemmEpi ep{ctx->b_mod, ctx->mod, ctx->Nmod, nullptr, 0, 1};
        CUDA_OK(launch_gemm(s, ctx->tm_csilu, ctx->tm_wmod, crows, ctx->Nmod, D, EPI_BIAS_F32, 0, ep));
        ctx->launches++;
    }
    const int ps = ctx->d.patch_size;
    if (ps == 2) {
        patch_embed_kernel<<<(M + 7) / 8, 256, 0, s>>>(x, x_rows, ctx->pe_w, ctx->pe_b, ctx->pos, ctx->x_tok, D, ctx->G,
                                                       ctx->C, M);
    } else {
        const int smem = 8 * ctx->C * ps * ps * (int)sizeof(float);
        patch_embed_generic_kernel<<<(M + 7) / 8, 256, smem, s>>>(x, x_rows, ctx->pe_w, ctx->pe_b, ctx->pos, ctx->x_tok, D,
                                                                  ctx->G, ctx->C, ps, M);
    }
    LAUNCH_OK();
    // L2 zig-zag (LFM_ZIGZAG): consecutive kernels sweep the token rows in opposite directions, so each starts on the
    // rows its producer wrote last (still L2-resident) instead of the rows that were evicted first.
    const int zig = ctx->zigzag;
    int dir = 1;  // patch_embed wrote x_tok upwards
    auto next_dir = [&]() {
        const int d = zig ? dir : 0;
        dir ^= 1;
        return d;
    };
    for (int l = 0; l < L; ++l) {
        BlockW& b = ctx->blk[l];
        const float* mb = ctx->mod + (size_t)l * 6 * D;  // shift_msa | scale_msa | gate_msa | shift_mlp | scale_mlp | gate_mlp
        {
            const int d = next_dir();
            CUDA_OK(launch_ln(s, ctx->x_tok, ctx->xn, mb, mb + D, Nmod, T, M, D, (zig ? 1 + d : 0) | (ctx->l2_hint ? 4 : 0)));
            ctx->launches++;
        }
        {
            GemmEpi ep{b.b_qkv, ctx->qkv, 3 * Dq, nullptr, 0, T};
            ep.reverse_m = next_dir();
            CUDA_OK(launch_gemm(s, ctx->tm_xn, b.tm_qkv, M, 3 * Dq, D, EPI_BIAS_BF16, 0, ep));
            ctx->launches++;
        }
        {
            next_dir();  // attention reads each (sample, head) once: the sweep direction only keeps the GEMMs alternating
            // head_dim 64 keeps the kernel's own ch^-1/2; the padded DiT-XL heads pass the true head_dim^-1/2
            const float sc = 1.4426950408889634f / sqrtf(static_cast<float>(ctx->dh));
            if (!ctx->qkv_head_major)                          // 256 tokens, head_dim 64: TMA + wgmma
                CUDA_OK(launch_attention_wgmma(s, ctx->tm_qkv_attn, ctx->attn, Dq, ctx->H, rows));
            else if (T == 16 || T == 64)                       // 4 x 4 / 8 x 8 token grids: the whole sequence in registers
                CUDA_OK(launch_attention_mma(s, ctx->qkv, ctx->attn, T, ctx->dhp, Dq, ctx->H, rows * ctx->H, ctx->dh == 64 ? 0.f : sc));
            else                                               // 1024 tokens, head_dim 72: keys streamed in chunks of 64
                CUDA_OK(launch_attention_flash(s, ctx->qkv, ctx->attn, T, ctx->dhp, Dq, ctx->H, rows * ctx->H, sc, false));
            ctx->launches++;
        }
        {
            GemmEpi ep{b.b_proj, ctx->x_tok, D, mb + 2 * D, Nmod, T};  // x += gate_msa * proj(...)   (models/DiT.py:129)
            ep.reverse_m = next_dir();
            CUDA_OK(launch_gemm(s, ctx->tm_attn, b.tm_proj, M, D, Dq, EPI_GATE_RESID_F32, 0, ep));
            ctx->launches++;
        }
        {
            const int d = next_dir();
            CUDA_OK(launch_ln(s, ctx->x_tok, ctx->xn, mb + 3 * D, mb + 4 * D, Nmod, T, M, D, (zig ? 1 + d : 0) | (ctx->l2_hint ? 4 : 0)));
            ctx->launches++;
        }
        {
            GemmEpi ep{b.b_fc1, ctx->hmid, Hd, nullptr, 0, T};
            ep.reverse_m = next_dir();
            CUDA_OK(launch_gemm(s, ctx->tm_xn, b.tm_fc1, M, Hd, D, EPI_BIAS_GELU_BF16, 0, ep));
            ctx->launches++;
        }
        {
            GemmEpi ep{b.b_fc2, ctx->x_tok, D, mb + 5 * D, Nmod, T};  // x += gate_mlp * fc2(...)   (models/DiT.py:130)
            ep.reverse_m = next_dir();
            CUDA_OK(launch_gemm(s, ctx->tm_hmid, b.tm_fc2, M, D, Hd, EPI_GATE_RESID_F32, 0, ep));
            ctx->launches++;
        }
    }
    {
        const float* mf = ctx->mod + (size_t)6 * L * D;  // shift | scale
        static DevOnce once;
        const int smem = 16 * D * (int)sizeof(float);
        CUDA_OK(smem_opt_in(once, final_layer_kernel, 16 * 1536 * 4));  // largest supported width (hidden_size <= 1536)
        int grid = (M + 7) / 8;
        if (grid > 2 * g_num_sms) grid = 2 * g_num_sms;
        if (ps == 2)
            final_layer_kernel<<<grid, 256, smem, s>>>(ctx->x_tok, mf, mf + D, Nmod, ctx->fin_w, ctx->fin_b, ctx->v_net, M, D,
                                                       ctx->G, ctx->C);
        else
            final_layer_generic_kernel<<<grid, 256, 0, s>>>(ctx->x_tok, mf, mf + D, Nmod, ctx->fin_w, ctx->fin_b, ctx->v_net, M,
                                                            D, ctx->G, ctx->C, ps);
        LAUNCH_OK();
    }
    return 0;
}

// Evaluate the (CFG-combined) velocity of n_img latents in `x` into `v_out` [n_img, C, H, W].
//   cfg_scale > 1: network batch = 2 n_img rows (labels y[0:n] conditional, y[n:2n] null), v = u + s (c - u).
static int eval_velocity(lfm_ctx* ctx, cudaStream_t s, const float* t, int t_numel, const float* x, int n_img,
                         const long long* y, float cfg_scale, float* v_out) {
    const size_t n = (size_t)n_img * ctx->chw;
    if (cfg_scale > 1.0f && ctx->arch == LFM_ARCH_UNET && ctx_unet_variant(ctx) == 0)
        return fail(ctx, "UNetModel has no forward_with_cfg (reference models/guided_diffusion/unet.py): cfg_scale must be <= 1");
    if (cfg_scale > 1.0f) {
        if (launch_network(ctx, s, t, t_numel, x, n_img, y, 2 * n_img)) return 1;
        cfg_combine_kernel<<<blocks_for(n), 256, 0, s>>>(ctx->v_net, v_out, n, cfg_scale, 0);
        LAUNCH_OK();
    } else {
        if (launch_network(ctx, s, t, t_numel, x, n_img, y, n_img)) return 1;
        CUDA_OK(cudaMemcpyAsync(v_out, ctx->v_net, n * sizeof(float), cudaMemcpyDeviceToDevice, s));
    }
    return 0;
}

static int check_ready(lfm_ctx* ctx, int rows, const char* who) {
    if (ctx == nullptr) return fail(ctx, "%s: null ctx", who);
    if (!ctx->finalized) return fail(ctx, "%s: lfm_finalize has not been called", who);
    if (rows < 1 || rows > ctx->max_rows)
        return fail(ctx, "%s: %d network rows requested, ctx finalized for %d", who, rows, ctx->max_rows);
    return 0;
}

extern "C" int lfm_forward(lfm_ctx* ctx, const float* t, int t_numel, const float* x, const int64_t* y, int B,
                           float cfg_scale, float* v_out, void* stream) {
    if (check_ready(ctx, B, "lfm_forward")) return 1;
    if (t == nullptr || x == nullptr || v_out == nullptr) return fail(ctx, "lfm_forward: null tensor");
    if (t_numel != 1 && t_numel != B) return fail(ctx, "lfm_forward: t has %d elements, expected 1 or %d", t_numel, B);
    CUDA_OK(cudaSetDevice(ctx->device));
    g_num_sms = ctx->num_sms;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const long long* yl = reinterpret_cast<const long long*>(y);
    if (cfg_scale > 1.0f && ctx->arch == LFM_ARCH_UNET && ctx_unet_variant(ctx) == 0)
        return fail(ctx, "lfm_forward: UNetModel has no forward_with_cfg; cfg_scale must be <= 1");
    if (cfg_scale > 1.0f) {
        if (B % 2 != 0) return fail(ctx, "lfm_forward: forward_with_cfg needs an even batch (got %d)", B);
        // a vector t has 2n entries in the reference; both halves carry the same times (the x halves are identical)
        const int n_img = B / 2;
        if (launch_network(ctx, s, t, t_numel, x, n_img, yl, B)) return 1;
        const size_t n = (size_t)n_img * ctx->chw;
        cfg_combine_kernel<<<blocks_for(n), 256, 0, s>>>(ctx->v_net, v_out, n, cfg_scale, 1);
        LAUNCH_OK();
    } else {
        if (launch_network(ctx, s, t, t_numel, x, B, yl, B)) return 1;
        CUDA_OK(cudaMemcpyAsync(v_out, ctx->v_net, (size_t)B * ctx->chw * sizeof(float), cudaMemcpyDeviceToDevice, s));
    }
    return 0;
}

// ------------------------------------------------------------------------------------------------
// fixed-step solvers: one captured graph per step kind, replayed from the host with no synchronisation

static int join_in(lfm_ctx* ctx, cudaStream_t user) {
    CUDA_OK(cudaEventRecord(ctx->ev_in, user));
    CUDA_OK(cudaStreamWaitEvent(ctx->stream, ctx->ev_in, 0));
    return 0;
}
static int join_out(lfm_ctx* ctx, cudaStream_t user) {
    CUDA_OK(cudaEventRecord(ctx->ev_out, ctx->stream));
    CUDA_OK(cudaStreamWaitEvent(user, ctx->ev_out, 0));
    return 0;
}

// body of one interval, recorded into ctx->stream (under capture or live)
static int record_step(lfm_ctx* ctx, int kind /*0 euler, 1 heun (with corrector)*/, int n_img, bool has_y, float cfg_scale) {
    cudaStream_t s = ctx->stream;
    const size_t n = (size_t)n_img * ctx->chw;
    const long long* y = has_y ? ctx->y_buf : nullptr;
    step_time_kernel<<<1, 32, 0, s>>>(ctx->t_grid, ctx->step_state, 0, ctx->t_eval);
    LAUNCH_OK();
    if (eval_velocity(ctx, s, ctx->t_eval, 1, ctx->x_state, n_img, y, cfg_scale, ctx->v_eff)) return 1;
    if (kind == 0) {
        euler_update_kernel<<<blocks_for(n), 256, 0, s>>>(ctx->x_state, ctx->v_eff, ctx->t_grid, ctx->step_state, n);
        LAUNCH_OK();
    } else {
        heun_predict_kernel<<<blocks_for(n), 256, 0, s>>>(ctx->x_state, ctx->v_eff, ctx->x_pred, ctx->t_grid,
                                                          ctx->step_state, n);
        LAUNCH_OK();
        step_time_kernel<<<1, 32, 0, s>>>(ctx->t_grid, ctx->step_state, 1, ctx->t_eval);
        LAUNCH_OK();
        if (eval_velocity(ctx, s, ctx->t_eval, 1, ctx->x_pred, n_img, y, cfg_scale, ctx->d_prime)) return 1;
        heun_correct_kernel<<<blocks_for(n), 256, 0, s>>>(ctx->x_state, ctx->v_eff, ctx->d_prime, ctx->x_pred, ctx->t_grid,
                                                          ctx->step_state, 1 << 30, n);
        LAUNCH_OK();
    }
    step_advance_kernel<<<1, 32, 0, s>>>(ctx->step_state);
    LAUNCH_OK();
    return 0;
}

static int get_step_graph(lfm_ctx* ctx, int kind, int n_img, bool has_y, float cfg_scale, cudaGraphExec_t* out,
                          int* launches) {
    char key[128];
    snprintf(key, sizeof(key), "k%d_n%d_y%d_c%.6f", kind, n_img, has_y ? 1 : 0, cfg_scale > 1.0f ? cfg_scale : 0.f);
    auto it = ctx->graphs.find(key);
    if (it != ctx->graphs.end()) {
        *out = it->second.exec;
        *launches = it->second.launches;
        return 0;
    }
    if (env_int("LFM_NO_GRAPH", 0)) {
        *out = nullptr;
        return 0;
    }
    // warm the lazily-set function attributes outside of capture
    const int64_t launches_before = ctx->launches;
    if (record_step(ctx, kind, n_img, has_y, cfg_scale)) return 1;
    CUDA_OK(cudaStreamSynchronize(ctx->stream));
    const int launches_per_replay = static_cast<int>(ctx->launches - launches_before);
    StepState zero{0, 0, 0};
    // (the warm-up advanced the device step counter and state; callers re-initialise both afterwards)
    cudaGraph_t graph = nullptr;
    CUDA_OK(cudaStreamBeginCapture(ctx->stream, cudaStreamCaptureModeThreadLocal));
    const int rc = record_step(ctx, kind, n_img, has_y, cfg_scale);
    cudaError_t e = cudaStreamEndCapture(ctx->stream, &graph);
    ctx->launches = launches_before;
    if (rc) return 1;
    if (e != cudaSuccess) return fail(ctx, "graph capture failed: %s", cudaGetErrorString(e));
    cudaGraphExec_t exec = nullptr;
    CUDA_OK(cudaGraphInstantiate(&exec, graph, 0));
    CUDA_OK(cudaGraphDestroy(graph));
    (void)zero;
    ctx->graphs[key].exec = exec;
    ctx->graphs[key].launches = launches_per_replay;
    *launches = launches_per_replay;
    *out = exec;
    return 0;
}

extern "C" int lfm_sample_fixed(lfm_ctx* ctx, int method, float* x_inout, const float* t_grid_host, int n_grid,
                                int t_as_vector, int heun_corrector_limit, const int64_t* y, int B_img, float cfg_scale,
                                lfm_ode_stats* stats, void* stream) {
    // bit 0 (t as a [B] vector): a vector of equal times and a 0-d time give the same conditioning vector - nothing to do
    const int perturb = (t_as_vector & LFM_FIXED_PERTURB) ? 1 : 0;
    if (perturb && method == LFM_METHOD_HEUN) return fail(ctx, "lfm_sample_fixed: perturb applies to the torchdiffeq grids (euler, midpoint, rk4)");
    const int rows = cfg_scale > 1.0f ? 2 * B_img : B_img;
    if (check_ready(ctx, rows, "lfm_sample_fixed")) return 1;
    if (method < LFM_METHOD_EULER || method > LFM_METHOD_RK4) return fail(ctx, "lfm_sample_fixed: unknown method %d", method);
    if (n_grid < 2 || n_grid > 8192) return fail(ctx, "lfm_sample_fixed: n_grid must be in [2, 8192] (got %d)", n_grid);
    if (x_inout == nullptr || t_grid_host == nullptr) return fail(ctx, "lfm_sample_fixed: null tensor");
    if (cfg_scale > 1.0f && y == nullptr) return fail(ctx, "lfm_sample_fixed: CFG needs labels");
    CUDA_OK(cudaSetDevice(ctx->device));
    g_num_sms = ctx->num_sms;
    cudaStream_t user = static_cast<cudaStream_t>(stream);
    const size_t n = (size_t)B_img * ctx->chw;
    const bool has_y = y != nullptr;

    if (method == LFM_METHOD_MIDPOINT || method == LFM_METHOD_RK4) {
        // torchdiffeq fixed-grid midpoint / rk4: the stage times of the whole trajectory are computed here in fp32
        // exactly as the Python expressions do (t0 + dt * (1/3) ...), uploaded once, and the stages are launched
        // back to back - no host synchronisation inside the loop.
        if (join_in(ctx, user)) return 1;
        cudaStream_t s = ctx->stream;
        const int n_int = n_grid - 1, S = method == LFM_METHOD_RK4 ? 4 : 2;
        if (n_int * S > 8192) return fail(ctx, "lfm_sample_fixed: too many stages (%d)", n_int * S);
        std::vector<float> tg(n_grid);
        CUDA_OK(cudaMemcpy(tg.data(), t_grid_host, n_grid * sizeof(float), cudaMemcpyDefault));
        std::vector<float> ts((size_t)n_int * S);
        const float third = (float)(1.0 / 3.0), two_thirds = (float)(2.0 / 3.0);
        for (int i = 0; i < n_int; ++i) {
            const float t0 = tg[i], t1 = tg[i + 1], dt = t1 - t0;
            // options["perturb"]: the first evaluation of a step one ulp past t0 (Perturb.NEXT), rk4's last one ulp before
            // t1 (Perturb.PREV) - in torchdiffeq's negated time; here in model time the directions flip
            const float t0e = perturb ? nextafterf(t0, t0 - 1.0f) : t0;
            if (S == 2) {
                ts[2 * i] = t0e;
                ts[2 * i + 1] = t0 + 0.5f * dt;
            } else {
                ts[4 * i] = t0e;
                ts[4 * i + 1] = t0 + dt * third;
                ts[4 * i + 2] = t0 + dt * two_thirds;
                ts[4 * i + 3] = perturb ? nextafterf(t1, t1 + 1.0f) : t1;
            }
        }
        CUDA_OK(cudaMemcpyAsync(ctx->t_grid, ts.data(), ts.size() * sizeof(float), cudaMemcpyHostToDevice, s));
        CUDA_OK(cudaMemcpyAsync(ctx->x_state, x_inout, n * sizeof(float), cudaMemcpyDeviceToDevice, s));
        const long long* yb = nullptr;
        if (has_y) {
            CUDA_OK(cudaMemcpyAsync(ctx->y_buf, y, (size_t)rows * sizeof(long long), cudaMemcpyDefault, s));
            yb = ctx->y_buf;
        }
        CUDA_OK(cudaStreamSynchronize(s));  // ts is host stack/heap memory
        float* y0 = ctx->x_state;
        float* ytmp = ctx->x_pred;
        float** k = ctx->kbuf;
        int64_t nfe = 0;
        for (int i = 0; i < n_int; ++i) {
            const float dt = tg[i + 1] - tg[i];
            const float* tp = ctx->t_grid + (size_t)i * S;
            if (S == 2) {
                if (eval_velocity(ctx, s, tp, 1, y0, B_img, yb, cfg_scale, k[0])) return 1;
                fixed_rk_stage_kernel<<<blocks_for(n), 256, 0, s>>>(0, y0, k[0], nullptr, nullptr, nullptr, 0.5f * dt, ytmp, n);
                LAUNCH_OK();
                if (eval_velocity(ctx, s, tp + 1, 1, ytmp, B_img, yb, cfg_scale, k[1])) return 1;
                fixed_rk_stage_kernel<<<blocks_for(n), 256, 0, s>>>(1, y0, nullptr, k[1], nullptr, nullptr, dt, y0, n);
                LAUNCH_OK();
            } else {
                if (eval_velocity(ctx, s, tp, 1, y0, B_img, yb, cfg_scale, k[0])) return 1;
                fixed_rk_stage_kernel<<<blocks_for(n), 256, 0, s>>>(2, y0, k[0], nullptr, nullptr, nullptr, dt, ytmp, n);
                LAUNCH_OK();
                if (eval_velocity(ctx, s, tp + 1, 1, ytmp, B_img, yb, cfg_scale, k[1])) return 1;
                fixed_rk_stage_kernel<<<blocks_for(n), 256, 0, s>>>(3, y0, k[0], k[1], nullptr, nullptr, dt, ytmp, n);
                LAUNCH_OK();
                if (eval_velocity(ctx, s, tp + 2, 1, ytmp, B_img, yb, cfg_scale, k[2])) return 1;
                fixed_rk_stage_kernel<<<blocks_for(n), 256, 0, s>>>(4, y0, k[0], k[1], k[2], nullptr, dt, ytmp, n);
                LAUNCH_OK();
                if (eval_velocity(ctx, s, tp + 3, 1, ytmp, B_img, yb, cfg_scale, k[3])) return 1;
                fixed_rk_stage_kernel<<<blocks_for(n), 256, 0, s>>>(5, y0, k[0], k[1], k[2], k[3], dt, y0, n);
                LAUNCH_OK();
            }
            nfe += S;
        }
        CUDA_OK(cudaMemcpyAsync(x_inout, y0, n * sizeof(float), cudaMemcpyDeviceToDevice, s));
        if (join_out(ctx, user)) return 1;
        if (stats != nullptr) {
            stats->nfe = nfe;
            stats->accepted = n_int;
            stats->rejected = 0;
        }
        return 0;
    }

    // build (or fetch) the step graphs first: the warm-up run clobbers the solver state
    cudaGraphExec_t g_euler = nullptr, g_heun = nullptr;
    const int n_int = n_grid - 1;
    const int n_heun = method == LFM_METHOD_HEUN ? (heun_corrector_limit < n_int ? (heun_corrector_limit < 0 ? 0 : heun_corrector_limit) : n_int) : 0;
    const bool graphs = !env_int("LFM_NO_GRAPH", 0);
    if (join_in(ctx, user)) return 1;
    int l_euler = 0, l_heun = 0;
    if (graphs) {
        if (n_heun < n_int && get_step_graph(ctx, 0, B_img, has_y, cfg_scale, &g_euler, &l_euler)) return 1;
        if (n_heun > 0 && get_step_graph(ctx, 1, B_img, has_y, cfg_scale, &g_heun, &l_heun)) return 1;
    }
    cudaStream_t s = ctx->stream;
    CUDA_OK(cudaMemcpyAsync(ctx->t_grid, t_grid_host, (size_t)n_grid * sizeof(float), cudaMemcpyDefault, s));
    CUDA_OK(cudaMemcpyAsync(ctx->x_state, x_inout, n * sizeof(float), cudaMemcpyDeviceToDevice, s));
    if (has_y) CUDA_OK(cudaMemcpyAsync(ctx->y_buf, y, (size_t)rows * sizeof(long long), cudaMemcpyDefault, s));
    StepState st0{0, n_int, perturb};
    CUDA_OK(cudaMemcpyAsync(ctx->step_state, &st0, sizeof(st0), cudaMemcpyHostToDevice, s));
    CUDA_OK(cudaStreamSynchronize(s));  // st0 / t_grid_host are host stack/pageable memory
    int64_t nfe = 0;
    for (int i = 0; i < n_int; ++i) {
        const int kind = i < n_heun ? 1 : 0;
        cudaGraphExec_t g = kind ? g_heun : g_euler;
        if (g != nullptr) {
            CUDA_OK(cudaGraphLaunch(g, s));
            ctx->launches += kind ? l_heun : l_euler;
        } else {
            if (record_step(ctx, kind, B_img, has_y, cfg_scale)) return 1;
        }
        nfe += kind ? 2 : 1;
    }
    CUDA_OK(cudaMemcpyAsync(x_inout, ctx->x_state, n * sizeof(float), cudaMemcpyDeviceToDevice, s));
    if (join_out(ctx, user)) return 1;
    if (stats != nullptr) {
        stats->nfe = nfe;
        stats->accepted = n_int;
        stats->rejected = 0;
    }
    return 0;
}

// ------------------------------------------------------------------------------------------------
// dopri5 (torchdiffeq semantics; SURVEY.md 8(c)).  Integrates s = -t upward with the field -v(-s, y).

static const double DP_ALPHA[6] = {1.0 / 5, 3.0 / 10, 4.0 / 5, 8.0 / 9, 1.0, 1.0};
static const double DP_BETA[6][6] = {
    {1.0 / 5, 0, 0, 0, 0, 0},
    {3.0 / 40, 9.0 / 40, 0, 0, 0, 0},
    {44.0 / 45, -56.0 / 15, 32.0 / 9, 0, 0, 0},
    {19372.0 / 6561, -25360.0 / 2187, 64448.0 / 6561, -212.0 / 729, 0, 0},
    {9017.0 / 3168, -355.0 / 33, 46732.0 / 5247, 49.0 / 176, -5103.0 / 18656, 0},
    {35.0 / 384, 0, 500.0 / 1113, 125.0 / 192, -2187.0 / 6784, 11.0 / 84},
};
static const double DP_CERR[7] = {35.0 / 384 - 1951.0 / 21600, 0, 500.0 / 1113 - 22642.0 / 50085, 125.0 / 192 - 451.0 / 720,
                                  -2187.0 / 6784 - -12231.0 / 42400, 11.0 / 84 - 649.0 / 6300, -1.0 / 60};
static const double DP_MID[7] = {6025192743.0 / 30085553152.0 / 2, 0, 51252292925.0 / 65400821598.0 / 2,
                                 -2691868925.0 / 45128329728.0 / 2, 187940372067.0 / 1594534317056.0 / 2,
                                 -1776094331.0 / 19743644256.0 / 2, 11237099.0 / 235043384.0 / 2};

// torchdiffeq's adaptive Runge-Kutta pairs (rk_common.RKAdaptiveStepsizeODESolver; SURVEY.md 8(c), oracle/solvers.py
// _TABLEAUS): n = number of stage evaluations per step (alpha entries), k_1 = f0 and k_{n+1} = f1 of the next step.
struct RkTableau {
    int n, order;
    double alpha[6], beta[6][6], c_sol[7], c_err[7], c_mid[7];
    bool fsal;  // y1 == the last stage's input (c_sol[:n] == beta[n-1], c_sol[n] == 0)
};
static RkTableau make_tableau(int method) {
    RkTableau t{};
    if (method == LFM_ADAPTIVE_DOPRI5) {
        t.n = 6;
        t.order = 5;
        t.fsal = true;
        for (int i = 0; i < 6; ++i) {
            t.alpha[i] = DP_ALPHA[i];
            for (int j = 0; j < 6; ++j) t.beta[i][j] = DP_BETA[i][j];
        }
        for (int j = 0; j < 6; ++j) t.c_sol[j] = DP_BETA[5][j];
        for (int j = 0; j < 7; ++j) {
            t.c_err[j] = DP_CERR[j];
            t.c_mid[j] = DP_MID[j];
        }
    } else if (method == LFM_ADAPTIVE_BOSH3) {  // Bogacki-Shampine 3(2)
        t.n = 3;
        t.order = 3;
        t.fsal = true;
        const double a[3] = {1.0 / 2, 3.0 / 4, 1.0};
        const double b[3][3] = {{1.0 / 2, 0, 0}, {0.0, 3.0 / 4, 0}, {2.0 / 9, 1.0 / 3, 4.0 / 9}};
        const double cs[4] = {2.0 / 9, 1.0 / 3, 4.0 / 9, 0.0};
        const double ce[4] = {2.0 / 9 - 7.0 / 24, 1.0 / 3 - 1.0 / 4, 4.0 / 9 - 1.0 / 3, -1.0 / 8};
        const double cm[4] = {0.0, 0.5, 0.0, 0.0};
        for (int i = 0; i < 3; ++i) {
            t.alpha[i] = a[i];
            for (int j = 0; j < 3; ++j) t.beta[i][j] = b[i][j];
        }
        for (int j = 0; j < 4; ++j) {
            t.c_sol[j] = cs[j];
            t.c_err[j] = ce[j];
            t.c_mid[j] = cm[j];
        }
    } else {  // LFM_ADAPTIVE_HEUN: Heun-Euler 2(1)
        t.n = 1;
        t.order = 2;
        t.fsal = false;
        t.alpha[0] = 1.0;
        t.beta[0][0] = 1.0;
        t.c_sol[0] = t.c_sol[1] = 0.5;
        t.c_err[0] = 0.5;
        t.c_err[1] = -0.5;
        t.c_mid[0] = 0.5;
    }
    return t;
}

struct Dopri {
    lfm_ctx* ctx;
    cudaStream_t s;
    int n_img;
    const long long* y;
    float cfg_scale;
    size_t n;
    int64_t nfe = 0;
    RkTableau tab{};
    int method = 0;
};

// k_out = -v(t = -s_time, y)   (model sees a 0-d fp32 time)
static int dp_func(Dopri& d, float s_time, const float* yv, float* k_out) {
    lfm_ctx* ctx = d.ctx;
    const float t = -s_time;
    set_scalar_kernel<<<1, 32, 0, d.s>>>(ctx->t_eval, t);  // by-value launch argument: no host synchronisation
    LAUNCH_OK();
    if (eval_velocity(ctx, d.s, ctx->t_eval, 1, yv, d.n_img, d.y, d.cfg_scale, k_out)) return 1;
    negate_kernel<<<blocks_for(d.n), 256, 0, d.s>>>(k_out, d.n);
    LAUNCH_OK();
    d.nfe++;
    return 0;
}

// rms(a - b) relative to atol + rtol * |y0| into ctx->ratio[slot] (no synchronisation)
static int dp_rms_launch(Dopri& d, const float* a, const float* b, const float* y0, float atol, float rtol, int slot) {
    lfm_ctx* ctx = d.ctx;
    RkPtrs kp;
    for (int j = 0; j < 7; ++j) kp.k[j] = ctx->kbuf[j];
    rms_ratio_partial_kernel<<<kRmsBlocks, 256, 0, d.s>>>(a, b, kp, RkCoef{}, y0, y0, atol, rtol, d.n, ctx->partial, nullptr);
    LAUNCH_OK();
    rms_finalize_kernel<<<1, 32, 0, d.s>>>(ctx->partial, kRmsBlocks, d.n, ctx->ratio + slot);
    LAUNCH_OK();
    return 0;
}
static int dp_fetch(Dopri& d, int count) {  // ctx->ratio[0..count) -> ctx->ratio_host, one synchronisation
    lfm_ctx* ctx = d.ctx;
    CUDA_OK(cudaMemcpyAsync(ctx->ratio_host, ctx->ratio, count * sizeof(float), cudaMemcpyDeviceToHost, d.s));
    CUDA_OK(cudaStreamSynchronize(d.s));
    return 0;
}

// One attempted Dormand-Prince step, recorded into ctx->stream (live or under capture).  Every number that changes from
// step to step (the stage coefficients dt * beta_ij, the six stage times, dt * c_err) is read from ctx->dp_dev, and the
// buffers are fixed (an accepted step COPIES y1 -> y0 and k7 -> k1 instead of swapping pointers), so one captured
// graph serves the whole integration: per attempted step the host uploads 300 bytes, launches one graph and reads
// back one float.
static int dp_record_step(Dopri& d, float atol, float rtol) {
    lfm_ctx* ctx = d.ctx;
    cudaStream_t s = d.s;
    const size_t n = d.n;
    RkPtrs kp;
    for (int j = 0; j < 7; ++j) kp.k[j] = ctx->kbuf[j];
    float* y0 = ctx->x_state;
    float* y1 = ctx->x_pred;
    float* ytmp = ctx->y_stage;
    const int ns = d.tab.n;
    for (int i = 0; i < ns; ++i) {
        float* yi = (i == ns - 1 && d.tab.fsal) ? y1 : ytmp;
        rk_combine_dev_kernel<<<blocks_for(n), 256, 0, s>>>(y0, kp, i + 1, ctx->dp_dev->coef[i], yi, n);
        LAUNCH_OK();
        if (eval_velocity(ctx, s, ctx->dp_dev->t + i, 1, yi, d.n_img, d.y, d.cfg_scale, ctx->kbuf[i + 1])) return 1;
        negate_kernel<<<blocks_for(n), 256, 0, s>>>(ctx->kbuf[i + 1], n);
        LAUNCH_OK();
    }
    if (!d.tab.fsal) {  // y1 = y0 + dt * sum_j c_sol[j] k_j  (coefficient row ns of the step block)
        rk_combine_dev_kernel<<<blocks_for(n), 256, 0, s>>>(y0, kp, ns + 1, ctx->dp_dev->coef[ns], y1, n);
        LAUNCH_OK();
    }
    rms_ratio_partial_kernel<<<kRmsBlocks, 256, 0, s>>>(nullptr, nullptr, kp, RkCoef{}, y0, y1, atol, rtol, n, ctx->partial,
                                                        ctx->dp_dev->cerr);
    LAUNCH_OK();
    rms_finalize_kernel<<<1, 32, 0, s>>>(ctx->partial, kRmsBlocks, n, ctx->ratio);
    LAUNCH_OK();
    CUDA_OK(cudaMemcpyAsync(ctx->ratio_host, ctx->ratio, sizeof(float), cudaMemcpyDeviceToHost, s));
    return 0;
}

static int dp_get_graph(Dopri& d, float atol, float rtol, cudaGraphExec_t* out, int* launches) {
    lfm_ctx* ctx = d.ctx;
    char key[160];
    snprintf(key, sizeof(key), "dp%d_n%d_y%d_c%.6f_a%.9g_r%.9g", d.method, d.n_img, d.y != nullptr ? 1 : 0,
             d.cfg_scale > 1.0f ? d.cfg_scale : 0.f, atol, rtol);
    auto it = ctx->graphs.find(key);
    if (it != ctx->graphs.end()) {
        *out = it->second.exec;
        *launches = it->second.launches;
        return 0;
    }
    *out = nullptr;
    *launches = 0;
    if (env_int("LFM_NO_GRAPH", 0)) return 0;
    // warm-up run outside of capture (lazily set function attributes); it only writes scratch: ytmp, y1, k2..k7, ratio
    const int64_t before = ctx->launches;
    if (dp_record_step(d, atol, rtol)) return 1;
    CUDA_OK(cudaStreamSynchronize(d.s));
    const int per = static_cast<int>(ctx->launches - before);
    cudaGraph_t graph = nullptr;
    CUDA_OK(cudaStreamBeginCapture(d.s, cudaStreamCaptureModeThreadLocal));
    const int rc = dp_record_step(d, atol, rtol);
    cudaError_t e = cudaStreamEndCapture(d.s, &graph);
    ctx->launches = before;
    if (rc) return 1;
    if (e != cudaSuccess) return fail(ctx, "dopri5 graph capture failed: %s", cudaGetErrorString(e));
    cudaGraphExec_t exec = nullptr;
    CUDA_OK(cudaGraphInstantiate(&exec, graph, 0));
    CUDA_OK(cudaGraphDestroy(graph));
    ctx->graphs[key].exec = exec;
    ctx->graphs[key].launches = per;
    *out = exec;
    *launches = per;
    return 0;
}

extern "C" int lfm_sample_dopri5(lfm_ctx* ctx, float* x_inout, double t0, double t1, double rtol, double atol,
                                 const int64_t* y, int B_img, float cfg_scale, lfm_ode_stats* stats, void* stream) {
    return lfm_sample_adaptive(ctx, LFM_ADAPTIVE_DOPRI5, x_inout, t0, t1, rtol, atol, y, B_img, cfg_scale, stats, stream);
}

extern "C" int lfm_sample_adaptive(lfm_ctx* ctx, int method, float* x_inout, double t0, double t1, double rtol, double atol,
                                   const int64_t* y, int B_img, float cfg_scale, lfm_ode_stats* stats, void* stream) {
    const int rows = cfg_scale > 1.0f ? 2 * B_img : B_img;
    if (check_ready(ctx, rows, "lfm_sample_adaptive")) return 1;
    if (method < LFM_ADAPTIVE_DOPRI5 || method > LFM_ADAPTIVE_HEUN) return fail(ctx, "lfm_sample_adaptive: unknown method %d", method);
    if (x_inout == nullptr) return fail(ctx, "lfm_sample_adaptive: null tensor");
    if (!(t0 > t1)) return fail(ctx, "lfm_sample_adaptive: expects t0 > t1 (reference integrates t: 1 -> 0)");
    if (cfg_scale > 1.0f && y == nullptr) return fail(ctx, "lfm_sample_adaptive: CFG needs labels");
    CUDA_OK(cudaSetDevice(ctx->device));
    g_num_sms = ctx->num_sms;
    cudaStream_t user = static_cast<cudaStream_t>(stream);
    if (join_in(ctx, user)) return 1;
    Dopri d{ctx, ctx->stream, B_img, nullptr, cfg_scale, (size_t)B_img * ctx->chw};
    d.tab = make_tableau(method);
    d.method = method;
    const RkTableau& tab = d.tab;
    const int ns = tab.n;
    cudaStream_t s = d.s;
    const size_t n = d.n;
    if (y != nullptr) {
        CUDA_OK(cudaMemcpyAsync(ctx->y_buf, y, (size_t)rows * sizeof(long long), cudaMemcpyDefault, s));
        d.y = ctx->y_buf;
    }
    float* y0 = ctx->x_state;
    float* y1 = ctx->x_pred;
    float* ytmp = ctx->y_stage;
    float** k = ctx->kbuf;
    const float atol_f = (float)atol, rtol_f = (float)rtol;
    RkPtrs kp;
    for (int j = 0; j < 7; ++j) kp.k[j] = k[j];

    // the step graph first: its warm-up run scribbles over the scratch buffers (never over y0 / k1, set below)
    cudaGraphExec_t g_step = nullptr;
    int l_step = 0;
    CUDA_OK(cudaMemsetAsync(ctx->dp_dev, 0, sizeof(DpStep), s));
    if (dp_get_graph(d, atol_f, rtol_f, &g_step, &l_step)) return 1;

    CUDA_OK(cudaMemcpyAsync(y0, x_inout, n * sizeof(float), cudaMemcpyDeviceToDevice, s));
    double s0 = -t0;
    const double s_end = -t1;
    // _before_integrate: f0 and the initial step (_select_initial_step with order - 1); two synchronisations
    if (dp_func(d, (float)s0, y0, k[0])) return 1;
    if (dp_rms_launch(d, y0, nullptr, y0, atol_f, rtol_f, 0)) return 1;
    if (dp_rms_launch(d, k[0], nullptr, y0, atol_f, rtol_f, 1)) return 1;
    if (dp_fetch(d, 2)) return 1;
    const float d0 = ctx->ratio_host[0], d1 = ctx->ratio_host[1];
    float h0 = (d0 < 1e-5f || d1 < 1e-5f) ? 1e-6f : 0.01f * d0 / d1;
    h0 = fabsf(h0);
    axpy_kernel<<<blocks_for(n), 256, 0, s>>>(y0, k[0], h0, ytmp, n);
    LAUNCH_OK();
    if (dp_func(d, (float)(s0 + (double)h0), ytmp, k[1])) return 1;
    if (dp_rms_launch(d, k[1], k[0], y0, atol_f, rtol_f, 0)) return 1;
    if (dp_fetch(d, 1)) return 1;
    const float d2 = fabsf(ctx->ratio_host[0] / h0);
    float h1;
    if (d1 <= 1e-15f && d2 <= 1e-15f)
        h1 = fmaxf(1e-6f, h0 * 1e-3f);
    else
        h1 = powf(0.01f / fmaxf(d1, d2), 1.0f / (float)tab.order);
    double dt = (double)fminf(100.f * h0, fabsf(h1));

    double s_hi = s0;
    int64_t accepted = 0, rejected = 0;
    bool have_interp = false;
    while (s_end > s_hi) {
        if (accepted + rejected > 100000) return fail(ctx, "lfm_sample_adaptive: step limit exceeded");
        const double t0s = s_hi, t1s = t0s + dt;
        const float t0_32 = (float)t0s, dt_32 = (float)dt, t1_32 = (float)t1s;
        DpStep* hp = ctx->dp_host;  // the previous step's upload has completed: every step ends with a synchronisation
        memset(hp, 0, sizeof(DpStep));
        for (int i = 0; i < ns; ++i) {
            for (int j = 0; j <= i; ++j) hp->coef[i][j] = (float)tab.beta[i][j] * dt_32;
            const float si = tab.alpha[i] == 1.0 ? nextafterf(t1_32, t1_32 - 1.0f) : t0_32 + (float)tab.alpha[i] * dt_32;
            hp->t[i] = -si;
        }
        if (!tab.fsal)
            for (int j = 0; j <= ns; ++j) hp->coef[ns][j] = (float)tab.c_sol[j] * dt_32;
        for (int j = 0; j <= ns; ++j) hp->cerr[j] = dt_32 * (float)tab.c_err[j];
        CUDA_OK(cudaMemcpyAsync(ctx->dp_dev, hp, sizeof(DpStep), cudaMemcpyHostToDevice, s));
        if (g_step != nullptr) {
            CUDA_OK(cudaGraphLaunch(g_step, s));
            ctx->launches += l_step;
        } else if (dp_record_step(d, atol_f, rtol_f)) {
            return 1;
        }
        CUDA_OK(cudaStreamSynchronize(s));  // the ONE synchronisation of the step: the controller runs on the host in fp64
        d.nfe += ns;
        const float ratio = fabsf(ctx->ratio_host[0]);
        const bool accept = ratio <= 1.0f;
        if (accept) {
            accepted++;
            s_hi = t1s;
            if (t1s >= s_end) {
                // last step: evaluate the quartic dense output at s_end and finish
                RkCoef cm{};
                for (int j = 0; j <= ns; ++j) cm.c[j] = dt_32 * (float)tab.c_mid[j];
                const float xq = (float)((s_end - t0s) / (t1s - t0s));
                RkPtrs kq = kp;
                kq.k[6] = k[ns];  // the interpolant's f1 is the LAST stage derivative (slot 6 of the kernel's argument)
                dopri_interp_kernel<<<blocks_for(n), 256, 0, s>>>(y0, y1, kq, cm, dt_32, xq, ytmp, n);
                LAUNCH_OK();
                have_interp = true;
                break;
            }
            dp_accept_kernel<<<blocks_for(n), 256, 0, s>>>(y0, y1, k[0], k[ns], n);  // y0 <- y1, f0 <- the last stage derivative
            LAUNCH_OK();
        } else {
            rejected++;
        }
        double factor;
        if (ratio == 0.f) {
            factor = 10.0;
        } else {
            const double dfactor = ratio < 1.f ? 1.0 : 0.2;
            factor = fmin(10.0, fmax(0.9 / pow((double)ratio, 1.0 / (double)tab.order), dfactor));
        }
        dt = dt * factor;
    }
    if (!have_interp) return fail(ctx, "lfm_sample_adaptive: integration produced no step");
    CUDA_OK(cudaMemcpyAsync(x_inout, ytmp, n * sizeof(float), cudaMemcpyDeviceToDevice, s));
    if (join_out(ctx, user)) return 1;
    if (stats != nullptr) {
        stats->nfe = d.nfe;
        stats->accepted = accepted;
        stats->rejected = rejected;
    }
    return 0;
}

// ------------------------------------------------------------------------------------------------

extern "C" const char* lfm_last_error(const lfm_ctx* ctx) {
    if (ctx != nullptr && !ctx->err.empty()) return ctx->err.c_str();
    return g_last_error.c_str();
}

extern "C" int64_t lfm_launch_count(const lfm_ctx* ctx) { return ctx != nullptr ? ctx->launches : 0; }

extern "C" void lfm_destroy(lfm_ctx* ctx) {
    if (ctx == nullptr) return;
    cudaSetDevice(ctx->device);
    cudaDeviceSynchronize();
    for (auto& g : ctx->graphs)
        if (g.second.exec != nullptr) cudaGraphExecDestroy(g.second.exec);
    for (void* p : ctx->allocs) cudaFree(p);
    if (ctx->staging != nullptr) cudaFree(ctx->staging);
    delete ctx->un;
    if (ctx->ratio_host != nullptr) cudaFreeHost(ctx->ratio_host);
    if (ctx->dp_host != nullptr) cudaFreeHost(ctx->dp_host);
    if (ctx->stream != nullptr) cudaStreamDestroy(ctx->stream);
    if (ctx->ev_in != nullptr) cudaEventDestroy(ctx->ev_in);
    if (ctx->ev_out != nullptr) cudaEventDestroy(ctx->ev_out);
    delete ctx;
}

// ------------------------------------------------------------------------------------------------
// kernel-level test entry points

extern "C" int lfm_dbg_gemm(const void* a_bf16, const void* w_bf16, const float* bias, void* out, const float* gate,
                            int gate_stride, int rows_per_sample, int M, int N, int K, int epi, int block_n,
                            void* stream) {
    lfm_ctx* ctx = nullptr;
    if (K % 64 != 0 || N % 8 != 0) return fail(ctx, "lfm_dbg_gemm: K must be a multiple of 64 and N of 8");
    if (epi < EPI_BIAS_BF16 || epi > EPI_BIAS_F32) return fail(ctx, "lfm_dbg_gemm: unknown epilogue %d", epi);
    if (block_n != 0 && block_n != 128 && block_n != 256 && block_n != 512 && block_n != 640 && block_n != 1024)
        return fail(ctx, "lfm_dbg_gemm: block_n must be 0, 128, 256, 512, 640 or 1024");
    g_num_sms = query_num_sms();
    if (g_num_sms <= 0) return fail(ctx, "no CUDA device");
    CUtensorMap ta, tb;
    if (!make_tmap_bf16(&ta, a_bf16, M, K, kGemmBoxRows) || !make_tmap_bf16(&tb, w_bf16, N, K, kGemmBoxRows))
        return fail(ctx, "lfm_dbg_gemm: tensor map encode failed");
    GemmEpi ep{bias, out, N, gate, gate_stride, rows_per_sample > 0 ? rows_per_sample : 1};
    CUDA_OK(launch_gemm(static_cast<cudaStream_t>(stream), ta, tb, M, N, K, epi, block_n == 128 || block_n == 256 ? block_n : 0, ep));
    return 0;
}

extern "C" int lfm_dbg_attention(const void* qkv_bf16, void* out_bf16, int B, int H, int variant, float* dbg_s,
                                 void* stream) {
    lfm_ctx* ctx = nullptr;
    if (variant != 0 && variant != 1) return fail(ctx, "lfm_dbg_attention: variant must be 0 (wgmma) or 1 (mma.sync flash)");
    if (dbg_s != nullptr) return fail(ctx, "lfm_dbg_attention: dbg_s is not supported (pass NULL)");
    g_num_sms = query_num_sms();
    if (g_num_sms <= 0) return fail(ctx, "no CUDA device");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (variant == 0) {
        CUtensorMap tq;
        if (!make_tmap_bf16(&tq, qkv_bf16, (uint64_t)B * 256, (uint64_t)3 * H * 64, kGemmBoxRows))
            return fail(ctx, "lfm_dbg_attention: tensor map encode failed");
        CUDA_OK(launch_attention_wgmma(s, tq, static_cast<__nv_bfloat16*>(out_bf16), H * 64, H, B));
    } else {
        const float sc = 0.125f * 1.4426950408889634f;  // head_dim^-0.5 * log2(e), head_dim = 64
        CUDA_OK(launch_attention_flash(s, static_cast<const __nv_bfloat16*>(qkv_bf16), static_cast<__nv_bfloat16*>(out_bf16), 256, 64,
                                       H * 64, H, B * H, sc, true));
    }
    return 0;
}

extern "C" int lfm_dbg_attention_mma(const void* qkv_bf16, void* out_bf16, int B, int H, int T, int ch, int head_dim, void* stream) {
    lfm_ctx* ctx = nullptr;
    g_num_sms = query_num_sms();
    if (g_num_sms <= 0) return fail(ctx, "no CUDA device");
    if (!(ch == 64 || ch == 80) || head_dim <= 0 || head_dim > ch) return fail(ctx, "lfm_dbg_attention_mma: ch must be 64 or 80, head_dim <= ch");
    const float sc = 1.4426950408889634f / sqrtf(static_cast<float>(head_dim));
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const __nv_bfloat16* q = static_cast<const __nv_bfloat16*>(qkv_bf16);
    __nv_bfloat16* o = static_cast<__nv_bfloat16*>(out_bf16);
    if (T == 16 || T == 64)
        CUDA_OK(launch_attention_mma(s, q, o, T, ch, H * ch, H, B * H, sc));
    else if (T > 0 && T % 64 == 0)
        CUDA_OK(launch_attention_flash(s, q, o, T, ch, H * ch, H, B * H, sc, false));
    else
        return fail(ctx, "lfm_dbg_attention_mma: T must be 16 or a multiple of 64 (got %d)", T);
    return 0;
}

extern "C" int lfm_dbg_tokens(lfm_ctx* ctx, float* out, int B) {
    if (check_ready(ctx, B, "lfm_dbg_tokens")) return 1;
    if (ctx->arch != LFM_ARCH_DIT) return fail(ctx, "lfm_dbg_tokens: DiT only");
    CUDA_OK(cudaMemcpy(out, ctx->x_tok, (size_t)B * ctx->T * ctx->D * sizeof(float), cudaMemcpyDefault));
    return 0;
}
