// lfm_b200 - C ABI (include/lfm_b200.h): context, parameter upload, DiT forward, ODE solvers.
// Single translation unit; build:  nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -shared ...
#include "../../include/lfm_b200.h"

#include <algorithm>
#include <array>
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

// One tensor map of `rank` dimensions (innermost first; strides in bytes, of dimensions 1 .. rank - 1) in the 128-byte swizzle of
// every GEMM operand and output staging buffer.
static bool encode_tmap(CUtensorMap* m, CUtensorMapDataType dtype, cuuint32_t rank, const void* base, const cuuint64_t* dims,
                        const cuuint64_t* strides, const cuuint32_t* box, const cuuint32_t* elem_strides) {
    EncodeTiledFn fn = get_encode_fn();
    return fn != nullptr && fn(m, dtype, rank, const_cast<void*>(base), dims, strides, box, elem_strides, CU_TENSOR_MAP_INTERLEAVE_NONE,
                               CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}
static const cuuint32_t kUnitStrides[4] = {1, 1, 1, 1};

// Row-major bf16 matrix [rows, cols] with a row pitch of ld elements (ld > cols: a column window of a wider matrix);
// box = 64 columns (one 128-byte swizzle row) x box_rows rows.
static bool make_tmap_bf16_ld(CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows) {
    const cuuint64_t dims[2] = {cols, rows}, strides[1] = {ld * 2};
    const cuuint32_t box[2] = {64, box_rows};
    return encode_tmap(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, base, dims, strides, box, kUnitStrides);
}
static bool make_tmap_bf16(CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols, uint32_t box_rows) {
    return make_tmap_bf16_ld(m, base, rows, cols, cols, box_rows);
}
// Row-major e4m3 matrix [rows, cols] (the FP8 GEMM operands): box = 128 columns (one 128-byte swizzle row) x box_rows rows.
static bool make_tmap_e4m3(CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols, uint32_t box_rows) {
    const cuuint64_t dims[2] = {cols, rows}, strides[1] = {cols};
    const cuuint32_t box[2] = {128, box_rows};
    return encode_tmap(m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, base, dims, strides, box, kUnitStrides);
}
// A GEMM operand [rows, cols] of element type Op (bf16 or e4m3, the launch_gemm<Op> operand), box rows kGemmBoxRows.
template <typename Op>
static bool make_tmap_operand(CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols) {
    if constexpr (std::is_same_v<Op, __nv_fp8_e4m3>) return make_tmap_e4m3(m, base, rows, cols, kGemmBoxRows);
    return make_tmap_bf16(m, base, rows, cols, kGemmBoxRows);
}
// GEMM output [rows, cols] (bf16, or fp32 when f32) with a row pitch of ld elements, for the TMA-store epilogue (GemmEpi::out_map):
// box = 128 bytes x kGemmOutRows rows in the 128-byte swizzle of the staging buffers.  False when the map cannot exist (base or
// pitch not a multiple of 16 bytes): such outputs keep the register stores.
static bool make_tmap_out(CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, bool f32) {
    const uint64_t es = f32 ? 4 : 2;
    if ((reinterpret_cast<uintptr_t>(base) & 15) != 0 || (ld * es) % 16 != 0) return false;
    const cuuint64_t dims[2] = {cols, rows}, strides[1] = {ld * es};
    const cuuint32_t box[2] = {static_cast<cuuint32_t>(128 / es), static_cast<cuuint32_t>(kGemmOutRows)};
    return encode_tmap(m, f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, base, dims, strides, box,
                       kUnitStrides);
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

// Launch with the programmatic-stream-serialization attribute: see pdl_wait() in common.cuh.
template <typename... KArgs, typename... Args>
static cudaError_t launch_k(void (*kern)(KArgs...), dim3 grid, unsigned block, size_t smem, cudaStream_t s, Args&&... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid;
    cfg.blockDim = dim3(block);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = s;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}
// ONLY for kernels that execute pdl_wait() before their first global-memory access.

template <int BN, int EPI, typename Op>
static cudaError_t launch_gemm_inst(cudaStream_t s, const CUtensorMap& ta, const CUtensorMap& tb, int M, int N, int K,
                                    const GemmEpi& ep, const ConvGeom& cg, int ksplit, int split_row_pitch) {
    static DevOnce once;
    auto kern = gemm_bf16_wgmma<BN, EPI, Op>;
    if (cudaError_t e = smem_opt_in(once, kern, GemmCfg<BN>::kSmemBytes)) return e;
    const int items = ((M + kGemmBlockM - 1) / kGemmBlockM) * ((N + BN - 1) / BN) * ksplit;
    const int grid = items < g_num_sms ? items : g_num_sms;
    const CUtensorMap& tc = ep.out_map != nullptr ? *ep.out_map : ta;  // unread without an out_map
    return launch_k(kern, dim3(grid), kGemmThreads, GemmCfg<BN>::kSmemBytes, s, ta, tb, tc, M, N, K, ep, cg, ksplit, split_row_pitch);
}

// Tile width: 256 columns, unless N fits in 128 or the 256-wide tiles would leave more than half of the SMs idle (small
// sampling batches) - then 128, which doubles the tiles of the launch.
static int pick_block_n(int M, int N) {
    const int tiles256 = ((M + kGemmBlockM - 1) / kGemmBlockM) * ((N + 255) / 256);
    return (N <= 128 || 2 * tiles256 <= g_num_sms) ? 128 : 256;
}

// A and W are tensor maps with a box of {64, kGemmBoxRows} (make_tmap_bf16 / make_tmap_act4d); block_n = 128 or 256
// (0: pick_block_n).  The batched GEMMs of ConvGeom need block_n 256 when N is a multiple of 256 (W rows of one group).
// Only plain 2-D GEMMs (no taps, no batching, no split-K) without GroupNorm statistics store through ep.out_map.
// Op = __nv_fp8_e4m3: e4m3 operands (make_tmap_e4m3 maps, ep.a_scale / ep.w_scale set), plain 2-D GEMMs with a bf16 epilogue
// only.  K is a multiple of gemm_block_k<Op>(): 64 for bf16, 128 for e4m3.
template <typename Op = __nv_bfloat16>
static cudaError_t launch_gemm(cudaStream_t s, const CUtensorMap& ta, const CUtensorMap& tb, int M, int N, int K, int epi,
                               int block_n, const GemmEpi& ep, const ConvGeom& cg = ConvGeom{0, 0, 0, 0, 1}, int ksplit = 1,
                               int split_row_pitch = 0) {
    if (block_n == 0) block_n = cg.batch_m > 0 ? 256 : pick_block_n(M, N);
    GemmEpi e = ep;
    if (cg.taps != 0 || cg.batch_m != 0 || ksplit != 1 || ep.gn_bins != nullptr) e.out_map = nullptr;
#define LFM_GEMM_CASE(BN, E) \
    if (block_n == BN && epi == E) return launch_gemm_inst<BN, E, Op>(s, ta, tb, M, N, K, e, cg, ksplit, split_row_pitch);
    if constexpr (std::is_same_v<Op, __nv_fp8_e4m3>) {
        if (cg.taps != 0 || cg.batch_m != 0 || ksplit != 1 || ep.gn_bins != nullptr || K % gemm_block_k<Op>() != 0)
            return cudaErrorInvalidValue;
        LFM_GEMM_CASE(256, EPI_BIAS_BF16)
        LFM_GEMM_CASE(256, EPI_BIAS_GELU_BF16)
        LFM_GEMM_CASE(128, EPI_BIAS_BF16)
        LFM_GEMM_CASE(128, EPI_BIAS_GELU_BF16)
    } else {
        LFM_GEMM_CASE(256, EPI_BIAS_BF16)
        LFM_GEMM_CASE(256, EPI_BIAS_GELU_BF16)
        LFM_GEMM_CASE(256, EPI_GATE_RESID_F32)
        LFM_GEMM_CASE(256, EPI_BIAS_F32)
        LFM_GEMM_CASE(128, EPI_BIAS_BF16)
        LFM_GEMM_CASE(128, EPI_BIAS_GELU_BF16)
        LFM_GEMM_CASE(128, EPI_GATE_RESID_F32)
        LFM_GEMM_CASE(128, EPI_BIAS_F32)
    }
#undef LFM_GEMM_CASE
    return cudaErrorInvalidValue;
}

template <int NV, typename OutT>
static cudaError_t launch_ln_inst(cudaStream_t s, const float* x, OutT* y, const float* shift, const float* scale, int mod_stride,
                                  int rows_per_sample, int M, int down, float* ys) {
    static DevOnce once;
    auto kern = ln_modulate_kernel<NV, OutT>;
    if (cudaError_t e = smem_opt_in(once, kern, ln_smem_bytes(NV))) return e;
    const int tiles = (M + kLnRows - 1) / kLnRows;
    const int grid = tiles < g_num_sms ? tiles : g_num_sms;
    return launch_k(kern, dim3(grid), kLnRows * 32, ln_smem_bytes(NV), s, x, y, shift, scale, mod_stride, rows_per_sample, M, down, ys);
}
// The widths ln_modulate_kernel is instantiated for (launch_ln's switch): D = 128 NV with NV in {2, 3, 6, 8, 9}, the hidden sizes
// 256, 384, 768, 1024 and 1152.
static bool ln_width_ok(int D) {
    const int nv = D / 128;
    return D % 128 == 0 && (nv == 2 || nv == 3 || nv == 6 || nv == 8 || nv == 9);
}
// A kLnRows-row tile must not straddle two samples (the DiT token counts are 16, 64, 256 and 1024).
static bool ln_rows_per_sample_ok(int rows_per_sample) { return rows_per_sample > 0 && rows_per_sample % kLnRows == 0; }

// down = 0 / 1: the grid sweeps the rows upwards / downwards (ln_modulate_kernel).  OutT = __nv_fp8_e4m3: e4m3 codes and their row
// scales ys [M] (NULL for bf16).
template <typename OutT>
static cudaError_t launch_ln(cudaStream_t s, const float* x, OutT* y, const float* shift, const float* scale, int mod_stride,
                             int rows_per_sample, int M, int D, int down, float* ys) {
    if (!ln_width_ok(D) || !ln_rows_per_sample_ok(rows_per_sample)) return cudaErrorInvalidValue;
    switch (D / 128) {
        case 2: return launch_ln_inst<2>(s, x, y, shift, scale, mod_stride, rows_per_sample, M, down, ys);
        case 3: return launch_ln_inst<3>(s, x, y, shift, scale, mod_stride, rows_per_sample, M, down, ys);
        case 6: return launch_ln_inst<6>(s, x, y, shift, scale, mod_stride, rows_per_sample, M, down, ys);
        case 8: return launch_ln_inst<8>(s, x, y, shift, scale, mod_stride, rows_per_sample, M, down, ys);
        case 9: return launch_ln_inst<9>(s, x, y, shift, scale, mod_stride, rows_per_sample, M, down, ys);
        default: return cudaErrorInvalidValue;
    }
}

// Patch sizes with a patch-embed and a final-layer kernel (launch_patch_embed, launch_final_layer): 2, and 4 or 8 on the generic ones.
static bool dit_patch_ok(int p) { return p == 2 || p == 4 || p == 8; }

// lfm_set_param's per-row e4m3 quantisation (quantize_rows_e4m3_kernel) of an fp32 weight [N, K] on the device.
static void launch_quantize_rows_e4m3(cudaStream_t s, const float* w, __nv_fp8_e4m3* codes, float* scales, int N, int K) {
    quantize_rows_e4m3_kernel<<<(N + 7) / 8, 256, 0, s>>>(w, codes, scales, N, K);
}

static inline unsigned blocks_for(size_t n, int threads = 256) { return static_cast<unsigned>((n + threads - 1) / threads); }

#include "attention_host.inc"

// ------------------------------------------------------------------------------------------------
// context

// What lfm_set_param makes of an fp32 source: a layout of its elements ...
enum class Layout {
    COPY,             // as given
    CONV,             // conv weight [Co, Ci, kh, kw] -> [Co, kh, kw, Ci]
    TRANSPOSE,        // [R, rest] -> [rest, R]
    QKV_W,            // qkv weight / bias rows re-ordered, qkv_src_row: aux = {head dim, its stored width, source order,
    QKV_B,            //   destination order}
    PROJ_PAD,         // DiT proj weight with zero columns for the padded head channels (aux = {head dim, its stored width})
    RESAMPLE_FILTER,  // the constant resample_filter of EDM.py:96-98: validated, not stored
};
// ... stored as one of these types.
enum class Store {
    F32,
    BF16,
    E4M3_ROWS,  // e4m3 codes with one fp32 scale per row (ParamSlot::row_scale): the FP8 mode's qkv and fc1 weights
};

struct ParamSlot {
    void* dst = nullptr;  // device destination
    std::vector<int64_t> shape;
    size_t numel = 0;
    Layout layout = Layout::COPY;
    Store store = Store::F32;
    std::array<int, 4> aux{};
    float* row_scale = nullptr;  // E4M3_ROWS: [rows of dst]
    bool set = false;
};

// The network a context runs: lfm_create's DiT, or one of the flavours of the UNet program (unet_host.inc, ctx->un): the two
// UNets, the VAE decoder (lfm_create_vae) and the VAE encoder (lfm_create_vae_encoder).
enum class NetKind { DIT, ADM, EDM, VAE, VAE_ENC };

struct BlockW {
    void *w_qkv, *w_fc1;                     // the LayerNorm-fed weights, in the operand type of the mode (with_ln_operand) ...
    float *s_qkv = nullptr, *s_fc1 = nullptr;  // ... and their per-row scales (NULL for bf16)
    __nv_bfloat16 *w_proj, *w_fc2;
    float *b_qkv, *b_proj, *b_fc1, *b_fc2;
    CUtensorMap tm_qkv, tm_proj, tm_fc1, tm_fc2;
};

struct UNetState;

// The conditioning stage of the DiT, ADM and EDM networks (kernels.cuh: timestep_features_kernel, condition_mlp_kernel): the
// timestep MLP W0 [E, feat] and W2 [E, E], the label table with its label rule, and every layer's modulation rows (the DiT's adaLN,
// the UNets' FiLM) concatenated into one weight [n_mod, E] for one GEMM.  cond_register, cond_finalize, cond_launch.
struct Conditioning {
    int feat = 0, E = 0;             // timestep-feature width and embedding width (E 0: the network has no stage)
    int max_row = 0, null_row = -1;  // condition_mlp_kernel's label rule
    int n_mod = 0, mod_rows = 0;     // rows of the modulation weight, and those registered so far (cond_add_mod)
    float *w0 = nullptr, *b0 = nullptr, *w2 = nullptr, *b2 = nullptr, *table = nullptr, *b_mod = nullptr;
    __nv_bfloat16* w_mod = nullptr;
    // workspace: tf [R, feat], h1 [R, E], c_silu [max(R, 128), E], mod [R, n_mod]
    float *tf = nullptr, *h1 = nullptr, *mod = nullptr;
    __nv_bfloat16* c_silu = nullptr;
    CUtensorMap tm_csilu, tm_wmod, tmo_mod;
};
// The K of both MLP layers (the feature width and E): condition_mlp_kernel reads a weight row as float4 per lane.  4096 is the widest
// E = 4 model_channels that lfm_create_unet / lfm_create_edm admit (2 max(channel_mult) model_channels <= 2048).
constexpr int kConditionMaxK = 4096;
static bool condition_k_ok(int K) { return K >= 128 && K % 128 == 0 && K <= kConditionMaxK; }

struct lfm_ctx {
    lfm_model_desc d{};
    NetKind net = NetKind::DIT;
    UNetState* un = nullptr;
    int device = 0;
    int num_sms = 0;
    int D = 0, L = 0, H = 0, T = 0, G = 0, C = 0, Hd = 0, HW = 0;
    int in_chw = 0, out_chw = 0;  // floats of one image of the network input / of the solver state and the velocity
    int dh = 64, dhp = 64, Dq = 0;  // head_dim, its stored (zero-padded) width and the width H * dhp of the attention tensors
    int max_rows = 0;
    bool fp8 = false;  // lfm_set_fp8: qkv and fc1 on e4m3 operands
    bool finalized = false;
    std::string err;
    int64_t launches = 0;

    std::unordered_map<std::string, ParamSlot> params;
    std::vector<void*> allocs;
    float* staging = nullptr;
    size_t staging_elems = 0;

    Conditioning cond;  // DiT, ADM and EDM

    // parameters
    float *pos = nullptr, *pe_w = nullptr, *pe_b = nullptr, *fin_w = nullptr, *fin_b = nullptr;
    std::vector<BlockW> blk;

    // workspace
    float *x_tok = nullptr, *v_net = nullptr;
    void* xn = nullptr;            // ln_modulate's output, in the operand type of the mode (with_ln_operand) ...
    float* xn_scale = nullptr;     // ... and its row scales (NULL for bf16)
    __nv_bfloat16 *qkv = nullptr, *attn = nullptr, *hmid = nullptr;
    CUtensorMap tm_xn, tm_attn, tm_hmid;
    CUtensorMap tmo_qkv, tmo_hmid, tmo_x_tok;  // GEMM outputs (make_tmap_out): the TMA-store epilogue
    AttnOp attn_op;  // qkv -> attn of every block

    // solver state
    cudaStream_t stream = nullptr;
    cudaEvent_t ev_in = nullptr, ev_out = nullptr;
    float *x_state = nullptr, *x_pred = nullptr, *t_grid = nullptr, *t_stage = nullptr, *t_eval = nullptr,
          *coef = nullptr, *ratio = nullptr, *y_stage = nullptr;
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

static size_t numel(const std::vector<int64_t>& shape) {
    size_t n = 1;
    for (int64_t v : shape) n *= static_cast<size_t>(v);
    return n;
}

static void add_param(lfm_ctx* ctx, const std::string& key, void* dst, std::vector<int64_t> shape, Layout layout = Layout::COPY,
                      Store store = Store::F32, std::array<int, 4> aux = {}, float* row_scale = nullptr) {
    ParamSlot s;
    s.dst = dst;
    s.numel = numel(shape);
    s.shape = std::move(shape);
    s.layout = layout;
    s.store = store;
    s.aux = aux;
    s.row_scale = row_scale;
    ctx->params[key] = s;
}

// A parameter whose storage holds exactly its registered shape: allocate numel(shape) elements and register them.
template <typename Tp>
static int alloc_param(lfm_ctx* ctx, const std::string& key, Tp** p, const std::vector<int64_t>& shape, Layout layout = Layout::COPY,
                       Store store = Store::F32, std::array<int, 4> aux = {}) {
    if (dev_alloc(ctx, p, numel(shape))) return 1;
    add_param(ctx, key, *p, shape, layout, store, aux);
    return 0;
}

// The conditioning stage's parameters.  w0 / w2: the key prefixes of the two Linear layers ("<prefix>weight", "<prefix>bias");
// table_key: the label table of table_rows labels (NULL: none), stored as given, [table_rows, E] (Layout::COPY), or transposed from a
// bias-free Linear on a one-hot, [E, table_rows], with one all-zero row appended after the labels (Layout::TRANSPOSE, EDM's map_label:
// the dropped label).  The label rule reads rows 0 .. max_row, the last label row (COPY) or the zero row (TRANSPOSE); null_row is
// the row of y == NULL (-1: no table term).  n_mod: rows of the modulation weight, registered by the layers with cond_add_mod.
static int cond_register(lfm_ctx* ctx, const std::string& w0, const std::string& w2, const char* table_key, int feat, int E,
                         int table_rows, Layout table_layout, int null_row, int n_mod) {
    Conditioning& c = ctx->cond;
    if (!condition_k_ok(feat) || !condition_k_ok(E))
        return fail(ctx, "conditioning: the feature width (%d) and the embedding width (%d) must be multiples of 128 up to %d", feat, E,
                    kConditionMaxK);
    c.feat = feat;
    c.E = E;
    c.n_mod = n_mod;
    c.max_row = table_layout == Layout::TRANSPOSE ? table_rows : table_rows - 1;
    c.null_row = null_row;
    if (alloc_param(ctx, w0 + "weight", &c.w0, {E, feat}) || alloc_param(ctx, w0 + "bias", &c.b0, {E}) ||
        alloc_param(ctx, w2 + "weight", &c.w2, {E, E}) || alloc_param(ctx, w2 + "bias", &c.b2, {E}))
        return 1;
    if (table_key != nullptr) {
        const bool zero_row = table_layout == Layout::TRANSPOSE;
        if (dev_alloc(ctx, &c.table, (size_t)(table_rows + zero_row) * E)) return 1;
        add_param(ctx, table_key, c.table, zero_row ? std::vector<int64_t>{E, table_rows} : std::vector<int64_t>{table_rows, E}, table_layout);
    }
    return dev_alloc(ctx, &c.w_mod, (size_t)n_mod * E) || dev_alloc(ctx, &c.b_mod, n_mod);
}
// Registers a layer's modulation Linear (prefix "weight" [rows, E], "bias" [rows]) as the next `rows` rows of the stage's modulation
// weight, and returns the offset of its rows in mod.
static int cond_add_mod(lfm_ctx* ctx, const std::string& prefix, int rows) {
    Conditioning& c = ctx->cond;
    const int off = c.mod_rows;
    add_param(ctx, prefix + "weight", c.w_mod + (size_t)off * c.E, {rows, c.E}, Layout::COPY, Store::BF16);
    add_param(ctx, prefix + "bias", c.b_mod + off, {rows});
    c.mod_rows += rows;
    return off;
}

// Releases one allocation of ctx->allocs (a parameter storage replaced before lfm_finalize).
static int dev_free(lfm_ctx* ctx, void* p) {
    if (p == nullptr) return 0;
    auto it = std::find(ctx->allocs.begin(), ctx->allocs.end(), p);
    if (it != ctx->allocs.end()) ctx->allocs.erase(it);
    CUDA_OK(cudaFree(p));
    return 0;
}

// Makes the context's device current and gives the launch helpers its SM count: the first step of every entry that uses the device.
static int bind(lfm_ctx* ctx) {
    CUDA_OK(cudaSetDevice(ctx->device));
    g_num_sms = ctx->num_sms;
    return 0;
}

// A context of `kind` on `device`, with its stream and both events.  The creators call it after their own shape checks, so a
// shape refusal never depends on the device.
static int new_ctx(const char* who, int device, NetKind kind, lfm_ctx** out) {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
        return fail(nullptr, "%s: no CUDA device (liblfm_b200 has no CPU path)", who);
    if (device < 0 || device >= ndev) return fail(nullptr, "%s: bad device %d", who, device);
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return fail(nullptr, "cudaGetDeviceProperties failed");
    if (prop.major != 9) return fail(nullptr, "%s: device %d is sm_%d%d; this library is sm_90a only", who, device, prop.major, prop.minor);
    lfm_ctx* ctx = new lfm_ctx();
    ctx->net = kind;
    ctx->device = device;
    ctx->num_sms = prop.multiProcessorCount;
    auto init = [&]() -> int {
        if (bind(ctx)) return 1;
        CUDA_OK(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
        CUDA_OK(cudaEventCreateWithFlags(&ctx->ev_in, cudaEventDisableTiming));
        CUDA_OK(cudaEventCreateWithFlags(&ctx->ev_out, cudaEventDisableTiming));
        return 0;
    };
    if (init()) {
        lfm_destroy(ctx);
        return 1;
    }
    *out = ctx;
    return 0;
}

// The creators' last step: hand out the context, or release it when building it failed (rc != 0).  The message stays
// available through lfm_last_error(NULL).
static int finish_create(lfm_ctx* ctx, int rc, lfm_ctx** out) {
    if (rc) {
        lfm_destroy(ctx);
        return 1;
    }
    *out = ctx;
    return 0;
}

// Storage and keys of block i's qkv and fc1 weights, the GEMMs whose A operand ln_modulate writes: bf16, or in FP8 mode (ctx->fp8)
// e4m3 codes with one fp32 scale per output channel, quantised from the fp32 source after the qkv re-order and head padding.
static int dit_register_ln_gemm_weights(lfm_ctx* ctx, int i) {
    BlockW& b = ctx->blk[i];
    const std::string p = "blocks." + std::to_string(i) + ".";
    const int D = ctx->D, Dq = ctx->Dq, Hd = ctx->Hd;
    const Store store = ctx->fp8 ? Store::E4M3_ROWS : Store::BF16;
    const size_t es = ctx->fp8 ? 1 : 2;
    uint8_t *qkv, *fc1;
    if (dev_alloc(ctx, &qkv, es * 3 * Dq * D) || dev_alloc(ctx, &fc1, es * Hd * D)) return 1;
    b.w_qkv = qkv;
    b.w_fc1 = fc1;
    b.s_qkv = b.s_fc1 = nullptr;
    if (store == Store::E4M3_ROWS && (dev_alloc(ctx, &b.s_qkv, 3 * Dq) || dev_alloc(ctx, &b.s_fc1, Hd))) return 1;
    const int layout = network_qkv_layout(ctx->T, ctx->dhp);
    add_param(ctx, p + "attn.qkv.weight", b.w_qkv, {3 * D, D}, layout == QKV_HEAD_MAJOR ? Layout::QKV_W : Layout::COPY, store,
              {ctx->dh, ctx->dhp, QKV_TIMM, layout}, b.s_qkv);
    add_param(ctx, p + "mlp.fc1.weight", b.w_fc1, {Hd, D}, Layout::COPY, store, {}, b.s_fc1);
    return 0;
}

// DiT parameter storage and state-dict keys.
static int dit_register(lfm_ctx* ctx) {
    const lfm_model_desc& d = ctx->d;
    const int D = ctx->D, L = ctx->L, Hd = ctx->Hd, T = ctx->T, Dq = ctx->Dq;
    const int ps = d.patch_size;
    const int P = ctx->C * ps * ps;  // elements of one patch = out-features of the final linear
    if (alloc_param(ctx, "pos_embed", &ctx->pos, {1, T, D}) ||
        alloc_param(ctx, "x_embedder.proj.weight", &ctx->pe_w, {D, 4, ps, ps}, Layout::TRANSPOSE) ||  // stored as [P, D]
        alloc_param(ctx, "x_embedder.proj.bias", &ctx->pe_b, {D}) ||
        alloc_param(ctx, "final_layer.linear.weight", &ctx->fin_w, {P, D}) ||
        alloc_param(ctx, "final_layer.linear.bias", &ctx->fin_b, {P}))
        return 1;
    // 256 frequencies (TimestepEmbedder, DiT.py:43-62); y NULL reads the last table row, the null class.  All adaLN modulation
    // layers in one table: block i at rows 6 i D, the final layer's after them.
    if (cond_register(ctx, "t_embedder.mlp.0.", "t_embedder.mlp.2.", "y_embedder.embedding_table.weight", 256, D, d.table_rows,
                      Layout::COPY, d.table_rows - 1, (6 * L + 2) * D))
        return 1;
    ctx->blk.resize(L);
    for (int i = 0; i < L; ++i) {
        BlockW& b = ctx->blk[i];
        const std::string p = "blocks." + std::to_string(i) + ".";
        // qkv and proj are stored with the padded head width dhp (Dq = H * dhp columns of attention output)
        if (dit_register_ln_gemm_weights(ctx, i)) return 1;
        if (dev_alloc(ctx, &b.b_qkv, 3 * Dq)) return 1;
        if (dev_alloc(ctx, &b.w_proj, (size_t)D * Dq)) return 1;
        const int layout = network_qkv_layout(T, ctx->dhp);
        add_param(ctx, p + "attn.qkv.bias", b.b_qkv, {3 * D}, layout == QKV_HEAD_MAJOR ? Layout::QKV_B : Layout::COPY, Store::F32,
                  {ctx->dh, ctx->dhp, QKV_TIMM, layout});
        add_param(ctx, p + "attn.proj.weight", b.w_proj, {D, D}, ctx->dhp != ctx->dh ? Layout::PROJ_PAD : Layout::COPY, Store::BF16,
                  {ctx->dh, ctx->dhp});
        if (alloc_param(ctx, p + "attn.proj.bias", &b.b_proj, {D}) ||
            alloc_param(ctx, p + "mlp.fc1.bias", &b.b_fc1, {Hd}) ||
            alloc_param(ctx, p + "mlp.fc2.weight", &b.w_fc2, {D, Hd}, Layout::COPY, Store::BF16) ||
            alloc_param(ctx, p + "mlp.fc2.bias", &b.b_fc2, {D}))
            return 1;
        cond_add_mod(ctx, p + "adaLN_modulation.1.", 6 * D);
    }
    cond_add_mod(ctx, "final_layer.adaLN_modulation.1.", 2 * D);
    return 0;
}

extern "C" int lfm_create(const lfm_model_desc* desc, int device, lfm_ctx** out) {
    lfm_ctx* ctx = nullptr;
    if (desc == nullptr || out == nullptr) return fail(nullptr, "lfm_create: null argument");
    if (desc->arch != LFM_ARCH_DIT) return fail(nullptr, "lfm_create: unsupported arch %d", desc->arch);
    // Geometries (models/DiT.py:355-415; img_resolution = image_size // f): patch 2 / 4 / 8 on latents whose token grid is
    // 4 x 4, 8 x 8, 16 x 16 or 32 x 32 - e.g. /2 on 32 x 32 (every released preset) or 64 x 64, /4 on 64 x 64 or 32 x 32, /8 on 32 x 32.
    if (!dit_patch_ok(desc->patch_size))
        return fail(nullptr, "lfm_create: patch_size must be 2, 4 or 8 (got %d)", desc->patch_size);
    {
        const int g = desc->img_resolution / desc->patch_size;
        if (desc->img_resolution <= 0 || desc->img_resolution % desc->patch_size != 0 || !(g == 4 || g == 8 || g == 16 || g == 32))
            return fail(nullptr, "lfm_create: the token grid (img_resolution / patch_size) must be 4, 8, 16 or 32 per side, i.e. 16, 64, "
                        "256 or 1024 tokens (got img_resolution %d, patch_size %d)", desc->img_resolution, desc->patch_size);
    }
    if (!ln_width_ok(desc->hidden_size))
        return fail(nullptr, "lfm_create: hidden_size must be one of 256, 384, 768, 1024, 1152 (got %d)", desc->hidden_size);
    if (desc->num_heads <= 0 || (desc->num_heads * 64 != desc->hidden_size && desc->num_heads * 72 != desc->hidden_size))
        return fail(nullptr, "lfm_create: head_dim must be 64 or 72 (hidden %d, heads %d)", desc->hidden_size, desc->num_heads);
    if (desc->mlp_hidden % 64 != 0) return fail(nullptr, "lfm_create: mlp_hidden must be a multiple of 64");
    if (desc->in_channels != 4) return fail(nullptr, "lfm_create: in_channels must be 4");
    if (new_ctx("lfm_create", device, NetKind::DIT, &ctx)) return 1;
    ctx->d = *desc;
    ctx->D = desc->hidden_size;
    ctx->L = desc->depth;
    ctx->H = desc->num_heads;
    ctx->G = desc->img_resolution / desc->patch_size;
    ctx->T = ctx->G * ctx->G;
    ctx->C = desc->in_channels;
    ctx->Hd = desc->mlp_hidden;
    ctx->HW = desc->img_resolution;
    ctx->in_chw = ctx->out_chw = ctx->C * ctx->HW * ctx->HW;
    // head_dim 72 (DiT-XL) is stored padded to 80 channels; the qkv rows are stored in network_qkv_layout's order
    ctx->dh = desc->hidden_size / desc->num_heads;
    ctx->dhp = ctx->dh == 72 ? 80 : 64;
    ctx->Dq = desc->num_heads * ctx->dhp;
    return finish_create(ctx, dit_register(ctx), out);
}

extern "C" int lfm_set_fp8(lfm_ctx* ctx, int enable) {
    if (ctx == nullptr) return fail(ctx, "lfm_set_fp8: null ctx");
    if (ctx->net != NetKind::DIT)
        return fail(ctx, "lfm_set_fp8: FP8 mode exists for the DiT only; this is a %s context",
                    ctx->net == NetKind::ADM ? "UNet" : ctx->net == NetKind::EDM ? "EDM" : "VAE");
    if (ctx->finalized) return fail(ctx, "lfm_set_fp8: the context is finalized; call it between lfm_create and lfm_finalize");
    const bool on = enable != 0;
    if (on == ctx->fp8) return 0;
    for (int i = 0; i < ctx->L; ++i)
        for (const char* w : {"attn.qkv.weight", "mlp.fc1.weight"}) {
            const std::string key = "blocks." + std::to_string(i) + "." + w;
            if (ctx->params[key].set)
                return fail(ctx, "lfm_set_fp8: %s was uploaded in the other mode; call lfm_set_fp8 before lfm_set_param", key.c_str());
        }
    if (bind(ctx)) return 1;
    ctx->fp8 = on;
    for (int i = 0; i < ctx->L; ++i) {
        BlockW& b = ctx->blk[i];
        if (dev_free(ctx, b.w_qkv) || dev_free(ctx, b.w_fc1) || dev_free(ctx, b.s_qkv) || dev_free(ctx, b.s_fc1) ||
            dit_register_ln_gemm_weights(ctx, i))
            return 1;
    }
    return 0;
}

// The matrix slot s's layout makes of its source, [rows, cols]: what E4M3_ROWS quantises row by row.
static std::pair<int, int> laid_out_dims(const ParamSlot& s) {
    const int r0 = static_cast<int>(s.shape[0]), rest = static_cast<int>(s.numel / r0);
    switch (s.layout) {
        case Layout::TRANSPOSE: return {rest, r0};
        case Layout::QKV_W: return {3 * (r0 / 3 / s.aux[0]) * s.aux[1], rest};  // 3 heads dhp rows
        case Layout::QKV_B: return {1, 3 * (r0 / 3 / s.aux[0]) * s.aux[1]};
        case Layout::PROJ_PAD: return {r0, r0 / s.aux[0] * s.aux[1]};  // heads dhp columns
        default: return {r0, rest};
    }
}

// Slot s's layout of the fp32 source src into out, [rows, cols] as bf16 (out_bf16) or fp32, on the default stream.  CONV and PROJ_PAD
// have bf16 kernels only, TRANSPOSE and QKV_B fp32 ones: cudaErrorInvalidValue for the other type.
static cudaError_t launch_layout(const ParamSlot& s, const float* src, void* out, bool out_bf16, int rows, int cols) {
    const size_t n = static_cast<size_t>(rows) * cols;
    const unsigned grid = blocks_for(n);
    const int r0 = static_cast<int>(s.shape[0]), K = static_cast<int>(s.numel / r0), dh = s.aux[0], dhp = s.aux[1];
    auto* ob = static_cast<__nv_bfloat16*>(out);
    auto* of = static_cast<float*>(out);
    switch (s.layout) {
        case Layout::COPY:
            if (!out_bf16) return cudaMemcpyAsync(of, src, n * sizeof(float), cudaMemcpyDeviceToDevice);
            f32_to_bf16_kernel<<<blocks_for((n + 3) / 4), 256>>>(src, ob, n);
            return cudaSuccess;
        case Layout::QKV_W:  // 3 heads dhp rows
            if (out_bf16) qkv_weight_reorder_kernel<<<grid, 256>>>(src, ob, K, r0 / 3 / dh, dh, dhp, s.aux[2], s.aux[3]);
            else qkv_weight_reorder_kernel<<<grid, 256>>>(src, of, K, r0 / 3 / dh, dh, dhp, s.aux[2], s.aux[3]);
            return cudaSuccess;
        case Layout::CONV:
            if (!out_bf16) break;
            conv_weight_repack_kernel<<<grid, 256>>>(src, ob, r0, static_cast<int>(s.shape[1]), static_cast<int>(s.shape[2] * s.shape[3]));
            return cudaSuccess;
        case Layout::PROJ_PAD:
            if (!out_bf16) break;
            dit_proj_weight_pad_kernel<<<grid, 256>>>(src, ob, r0, dh, dhp);
            return cudaSuccess;
        case Layout::TRANSPOSE:
            if (out_bf16) break;
            transpose_f32_kernel<<<grid, 256>>>(src, of, r0, K);
            return cudaSuccess;
        case Layout::QKV_B:
            if (out_bf16) break;
            qkv_bias_reorder_kernel<<<grid, 256>>>(src, of, r0 / 3 / dh, dh, dhp, s.aux[2], s.aux[3]);
            return cudaSuccess;
        case Layout::RESAMPLE_FILTER:
            break;
    }
    return cudaErrorInvalidValue;
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
    if (bind(ctx)) return 1;
    if (s.layout == Layout::COPY && s.store == Store::F32) {
        CUDA_OK(cudaMemcpy(s.dst, ptr, s.numel * sizeof(float), cudaMemcpyDefault));
        s.set = true;
        return 0;
    }
    // Every other transform reads the source from the staging buffer.  For E4M3_ROWS the layout writes fp32 behind the source,
    // and the rows of that matrix are quantised into the destination.
    const bool e4m3 = s.store == Store::E4M3_ROWS;
    const auto [rows, cols] = laid_out_dims(s);
    const size_t need = s.numel + (e4m3 ? static_cast<size_t>(rows) * cols : 0);
    if (ctx->staging_elems < need) {
        if (ctx->staging != nullptr) CUDA_OK(cudaFree(ctx->staging));
        ctx->staging = nullptr;
        CUDA_OK(cudaMalloc(&ctx->staging, need * sizeof(float)));
        ctx->staging_elems = need;
    }
    CUDA_OK(cudaMemcpy(ctx->staging, ptr, s.numel * sizeof(float), cudaMemcpyDefault));
    if (s.layout == Layout::RESAMPLE_FILTER) {
        float h[4] = {0.f, 0.f, 0.f, 0.f};
        CUDA_OK(cudaMemcpy(h, ctx->staging, sizeof(h), cudaMemcpyDeviceToHost));
        for (float v : h)
            if (v != 0.25f) return fail(ctx, "lfm_set_param(%s): resample_filter must be [[0.25, 0.25], [0.25, 0.25]] (EDM.py:96-98)", key);
    } else {
        float* laid = ctx->staging + s.numel;  // E4M3_ROWS only
        if (launch_layout(s, ctx->staging, e4m3 ? laid : s.dst, s.store == Store::BF16, rows, cols) != cudaSuccess)
            return fail(ctx, "lfm_set_param(%s): no kernel for this layout and storage type", key);
        if (e4m3) launch_quantize_rows_e4m3(nullptr, laid, static_cast<__nv_fp8_e4m3*>(s.dst), s.row_scale, rows, cols);
    }
    CUDA_OK(cudaGetLastError());
    CUDA_OK(cudaDeviceSynchronize());
    s.set = true;
    return 0;
}

static int alloc_solver_state(lfm_ctx* ctx, int R) {
    // solver state (sized for R latent rows)
    const size_t nst = (size_t)R * ctx->out_chw;
    if (dev_alloc(ctx, &ctx->x_state, nst)) return 1;
    if (dev_alloc(ctx, &ctx->x_pred, nst)) return 1;
    if (dev_alloc(ctx, &ctx->y_stage, nst)) return 1;
    for (int j = 0; j < 7; ++j)
        if (dev_alloc(ctx, &ctx->kbuf[j], nst)) return 1;
    if (dev_alloc(ctx, &ctx->t_grid, 8192 + 64)) return 1;
    if (dev_alloc(ctx, &ctx->t_stage, 2 * 8192)) return 1;  // S (n_grid - 1) stage times: Heun's 2 x 8191 at most
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

// The conditioning stage's workspace for R rows and its tensor maps.  c_silu, the modulation GEMM's A operand, has at least the
// 128 rows of one box.
static int cond_finalize(lfm_ctx* ctx, int R) {
    Conditioning& c = ctx->cond;
    const int Rpad = R < 128 ? 128 : R;
    if (dev_alloc(ctx, &c.tf, (size_t)R * c.feat) || dev_alloc(ctx, &c.h1, (size_t)R * c.E) || dev_alloc(ctx, &c.c_silu, (size_t)Rpad * c.E) ||
        dev_alloc(ctx, &c.mod, (size_t)R * c.n_mod))
        return 1;
    bool ok = make_tmap_bf16(&c.tm_csilu, c.c_silu, Rpad, c.E, kGemmBoxRows);
    ok &= make_tmap_bf16(&c.tm_wmod, c.w_mod, c.n_mod, c.E, kGemmBoxRows);
    ok &= make_tmap_out(&c.tmo_mod, c.mod, R, c.n_mod, c.n_mod, true);
    return ok ? 0 : fail(ctx, "lfm_finalize: cuTensorMapEncodeTiled failed (conditioning)");
}

// The element type of the DiT's LayerNorm-fed GEMM operands, xn and the qkv / fc1 weights: f(__nv_bfloat16{}), or in FP8 mode
// f(__nv_fp8_e4m3{}).  The one place lfm_finalize and the forward choose it.
template <typename F>
static int with_ln_operand(const lfm_ctx* ctx, F&& f) {
    return ctx->fp8 ? f(__nv_fp8_e4m3{}) : f(__nv_bfloat16{});
}

extern "C" int lfm_finalize(lfm_ctx* ctx, int max_batch) {
    if (ctx == nullptr) return fail(ctx, "lfm_finalize: null ctx");
    if (max_batch < 1) return fail(ctx, "lfm_finalize: max_batch must be >= 1");
    for (auto& kv : ctx->params)
        if (!kv.second.set) return fail(ctx, "lfm_finalize: missing key '%s' (strict)", kv.first.c_str());
    if (ctx->finalized && max_batch <= ctx->max_rows) return 0;
    if (ctx->finalized) return fail(ctx, "lfm_finalize: already finalized for %d rows; create a new ctx for %d", ctx->max_rows, max_batch);
    if (bind(ctx)) return 1;
    if (ctx->cond.E > 0 && cond_finalize(ctx, max_batch)) return 1;
    if (ctx->net != NetKind::DIT) {
        if (unet_finalize(ctx, max_batch)) return 1;
        if (alloc_solver_state(ctx, max_batch)) return 1;
        ctx->max_rows = max_batch;
        ctx->finalized = true;
        return 0;
    }
    const int D = ctx->D, Hd = ctx->Hd, T = ctx->T, R = max_batch, Dq = ctx->Dq;
    const size_t M = (size_t)R * T;
    if (dev_alloc(ctx, &ctx->x_tok, M * D)) return 1;
    // xn (with its row scales for e4m3) and the tensor maps of the LayerNorm-fed GEMMs' operands
    if (with_ln_operand(ctx, [&](auto op) {
            using Op = decltype(op);
            Op* xn = nullptr;
            if (dev_alloc(ctx, &xn, M * D) || (std::is_same_v<Op, __nv_fp8_e4m3> && dev_alloc(ctx, &ctx->xn_scale, M))) return 1;
            ctx->xn = xn;
            bool ok = make_tmap_operand<Op>(&ctx->tm_xn, xn, M, D);
            for (auto& b : ctx->blk)
                ok = ok && make_tmap_operand<Op>(&b.tm_qkv, b.w_qkv, 3 * Dq, D) && make_tmap_operand<Op>(&b.tm_fc1, b.w_fc1, Hd, D);
            return ok ? 0 : fail(ctx, "lfm_finalize: cuTensorMapEncodeTiled failed");
        }))
        return 1;
    if (dev_alloc(ctx, &ctx->qkv, M * 3 * Dq)) return 1;
    if (dev_alloc(ctx, &ctx->attn, M * Dq)) return 1;
    if (dev_alloc(ctx, &ctx->hmid, M * Hd)) return 1;
    if (dev_alloc(ctx, &ctx->v_net, (size_t)R * ctx->out_chw)) return 1;
    if (alloc_solver_state(ctx, R)) return 1;

    bool ok = make_tmap_bf16(&ctx->tm_attn, ctx->attn, M, Dq, kGemmBoxRows);
    ok &= make_tmap_bf16(&ctx->tm_hmid, ctx->hmid, M, Hd, kGemmBoxRows);
    ok &= attn_plan(&ctx->attn_op, ctx->qkv, ctx->attn, T, ctx->dhp, ctx->dh, ctx->H, network_qkv_layout(T, ctx->dhp), R);
    ok &= make_tmap_out(&ctx->tmo_qkv, ctx->qkv, M, 3 * Dq, 3 * Dq, false);
    ok &= make_tmap_out(&ctx->tmo_hmid, ctx->hmid, M, Hd, Hd, false);
    ok &= make_tmap_out(&ctx->tmo_x_tok, ctx->x_tok, M, D, D, true);
    for (auto& b : ctx->blk) {
        ok &= make_tmap_bf16(&b.tm_proj, b.w_proj, D, Dq, kGemmBoxRows);
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
#define COUNT_LAUNCH(call)                            \
    do {                                              \
        CUDA_OK(call);                                \
        ctx->launches++;                              \
    } while (0)
#define LAUNCH_K(...) COUNT_LAUNCH(launch_k(__VA_ARGS__))

static int check_ready(lfm_ctx* ctx, int rows, const char* who);

// The conditioning stage's kernels for `rows` rows (t_numel 1 broadcasts): tf [rows, feat], h1 = SiLU(w0 tf + b0) [rows, E] and
// c = SiLU(w2 h1 + b2 + table[row]) [rows, E] (bf16) with condition_mlp_kernel's label rule.  feat and E: condition_k_ok.
static int launch_condition(lfm_ctx* ctx, cudaStream_t s, const float* t, int t_numel, const long long* y, int rows, int feat, int E,
                            const float* w0, const float* b0, const float* w2, const float* b2, const float* table, int max_row,
                            int null_row, float* tf, float* h1, __nv_bfloat16* c) {
    LAUNCH_K(timestep_features_kernel, dim3(rows), 256, 0, s, t, t_numel, tf, feat);
    LAUNCH_K(condition_mlp_kernel<float>, dim3((E + 7) / 8), 256, 0, s, w0, b0, tf, rows, E, feat, nullptr, nullptr, 0, -1, h1);
    LAUNCH_K(condition_mlp_kernel<__nv_bfloat16>, dim3((E + 7) / 8), 256, 0, s, w2, b2, h1, rows, E, E, table, y, max_row, null_row, c);
    return 0;
}

// The conditioning stage for `rows` network rows, then every layer's modulation rows in one GEMM: mod = c W_mod^T + b_mod.  A 0-d t
// without labels (every unconditional preset) gives the same c for every row: one row is computed and all samples read it.
// *mod_stride: the stride between samples in mod for the reads of the modulation (n_mod, or 0 for that one row).
static int cond_launch(lfm_ctx* ctx, cudaStream_t s, const float* t, int t_numel, const long long* y, int rows, int* mod_stride) {
    const Conditioning& c = ctx->cond;
    const bool uniform = t_numel == 1 && y == nullptr;
    const int crows = uniform ? 1 : rows;
    *mod_stride = uniform ? 0 : c.n_mod;
    if (launch_condition(ctx, s, t, t_numel, y, crows, c.feat, c.E, c.w0, c.b0, c.w2, c.b2, c.table, c.max_row, c.null_row, c.tf, c.h1,
                         c.c_silu))
        return 1;
    GemmEpi ep{c.b_mod, c.mod, c.n_mod, nullptr, 0, 1};
    ep.out_map = &c.tmo_mod;
    COUNT_LAUNCH(launch_gemm(s, c.tm_csilu, c.tm_wmod, crows, c.n_mod, c.E, EPI_BIAS_F32, 0, ep));
    return 0;
}

#include "unet_host.inc"
#include "vae_host.inc"

// Patch embed of M token rows (T = G^2 per sample; row b reads latent b % x_rows): the specialised kernel for p = 2 (C = 4),
// the generic one, with its 8 patch vectors in dynamic shared memory, for p = 4 and 8.
static int launch_patch_embed(lfm_ctx* ctx, cudaStream_t s, const float* x, int x_rows, const float* Wt, const float* bias,
                              const float* pos, float* tok, int D, int G, int C, int p, int M) {
    if (p == 2) {
        patch_embed_kernel<<<(M + 7) / 8, 256, 0, s>>>(x, x_rows, Wt, bias, pos, tok, D, G, C, M);
    } else {
        const int smem = 8 * C * p * p * (int)sizeof(float);
        patch_embed_generic_kernel<<<(M + 7) / 8, 256, smem, s>>>(x, x_rows, Wt, bias, pos, tok, D, G, C, p, M);
    }
    LAUNCH_OK();
    return 0;
}

// FinalLayer + unpatchify of M token rows into v_net (NCHW fp32): the specialised kernel (16 x D weight in shared memory) for
// p = 2 (C = 4), the generic one for p = 4 and 8.  At most 2 blocks per SM; each warp loops over the rows beyond.
constexpr int kFinalLayerMaxD = 1536;  // widest D whose 16 x D weight fits the specialised kernel's shared memory (96 KB)
static int launch_final_layer(lfm_ctx* ctx, cudaStream_t s, const float* x, const float* shift, const float* scale, int mod_stride,
                              const float* W, const float* bias, float* v_net, int M, int D, int G, int C, int p) {
    static DevOnce once;
    CUDA_OK(smem_opt_in(once, final_layer_kernel, 16 * kFinalLayerMaxD * (int)sizeof(float)));
    int grid = (M + 7) / 8;
    if (grid > 2 * g_num_sms) grid = 2 * g_num_sms;
    if (p == 2)
        final_layer_kernel<<<grid, 256, 16 * D * (int)sizeof(float), s>>>(x, shift, scale, mod_stride, W, bias, v_net, M, D, G, C);
    else
        final_layer_generic_kernel<<<grid, 256, 0, s>>>(x, shift, scale, mod_stride, W, bias, v_net, M, D, G, C, p);
    LAUNCH_OK();
    return 0;
}

// x_whole: see run_unet_program (conditioned UNets only)
static int launch_network(lfm_ctx* ctx, cudaStream_t s, const float* t, int t_numel, const float* x, int x_rows,
                          const long long* y, int rows, bool x_whole) {
    if (ctx->net != NetKind::DIT) return launch_unet(ctx, s, t, t_numel, x, x_rows, y, rows, x_whole);
    const int D = ctx->D, L = ctx->L, Hd = ctx->Hd, T = ctx->T, Dq = ctx->Dq;
    const int M = rows * T;
    // c = t_emb(t) + y_emb(y) and every adaLN modulation vector of the network: mod [rows or 1, (6L+2) D]
    int Nmod = 0;  // stride between samples in the modulation table
    if (cond_launch(ctx, s, t, t_numel, y, rows, &Nmod)) return 1;
    const int ps = ctx->d.patch_size;
    if (launch_patch_embed(ctx, s, x, x_rows, ctx->pe_w, ctx->pe_b, ctx->pos, ctx->x_tok, D, ctx->G, ctx->C, ps, M)) return 1;
    // L2 zig-zag: consecutive kernels sweep the token rows in opposite directions, so each starts on the rows its
    // producer wrote last (still L2-resident) instead of the rows that were evicted first.
    int dir = 1;  // patch_embed wrote x_tok upwards
    auto next_dir = [&]() {
        const int d = dir;
        dir ^= 1;
        return d;
    };
    // LayerNorm + modulate of x_tok into xn, then the GEMM that reads xn (qkv, fc1), in the operand type of the mode
    auto ln_gemm = [&](const float* shift, const float* scale, const CUtensorMap& tw, const float* w_scale, int N, int epi, GemmEpi ep) {
        const int ln_dir = next_dir();
        ep.reverse_m = next_dir();
        ep.a_scale = ctx->xn_scale;
        ep.w_scale = w_scale;
        return with_ln_operand(ctx, [&](auto op) {
            using Op = decltype(op);
            COUNT_LAUNCH(launch_ln(s, ctx->x_tok, static_cast<Op*>(ctx->xn), shift, scale, Nmod, T, M, D, ln_dir, ctx->xn_scale));
            COUNT_LAUNCH(launch_gemm<Op>(s, ctx->tm_xn, tw, M, N, D, epi, 0, ep));
            return 0;
        });
    };
    for (int l = 0; l < L; ++l) {
        BlockW& b = ctx->blk[l];
        const float* mb = ctx->cond.mod + (size_t)l * 6 * D;  // shift_msa | scale_msa | gate_msa | shift_mlp | scale_mlp | gate_mlp
        {
            GemmEpi ep{b.b_qkv, ctx->qkv, 3 * Dq, nullptr, 0, T};
            ep.out_map = &ctx->tmo_qkv;
            if (ln_gemm(mb, mb + D, b.tm_qkv, b.s_qkv, 3 * Dq, EPI_BIAS_BF16, ep)) return 1;
        }
        {
            next_dir();  // attention reads each (sample, head) once: the sweep direction only keeps the GEMMs alternating
            COUNT_LAUNCH(launch_attention(ctx->attn_op, s, rows));
        }
        {
            GemmEpi ep{b.b_proj, ctx->x_tok, D, mb + 2 * D, Nmod, T};  // x += gate_msa * proj(...)   (models/DiT.py:129)
            ep.reverse_m = next_dir();
            ep.out_map = &ctx->tmo_x_tok;
            COUNT_LAUNCH(launch_gemm(s, ctx->tm_attn, b.tm_proj, M, D, Dq, EPI_GATE_RESID_F32, 0, ep));
        }
        {
            GemmEpi ep{b.b_fc1, ctx->hmid, Hd, nullptr, 0, T};
            ep.out_map = &ctx->tmo_hmid;
            if (ln_gemm(mb + 3 * D, mb + 4 * D, b.tm_fc1, b.s_fc1, Hd, EPI_BIAS_GELU_BF16, ep)) return 1;
        }
        {
            GemmEpi ep{b.b_fc2, ctx->x_tok, D, mb + 5 * D, Nmod, T};  // x += gate_mlp * fc2(...)   (models/DiT.py:130)
            ep.reverse_m = next_dir();
            ep.out_map = &ctx->tmo_x_tok;
            COUNT_LAUNCH(launch_gemm(s, ctx->tm_hmid, b.tm_fc2, M, D, Hd, EPI_GATE_RESID_F32, 0, ep));
        }
    }
    const float* mf = ctx->cond.mod + (size_t)6 * L * D;  // shift | scale
    return launch_final_layer(ctx, s, ctx->x_tok, mf, mf + D, Nmod, ctx->fin_w, ctx->fin_b, ctx->v_net, M, D, ctx->G, ctx->C, ps);
}

// Evaluate the (CFG-combined) velocity of n_img latents in `x` into `v_out` [n_img, C, H, W].
//   cfg_scale > 1: network batch = 2 n_img rows (labels y[0:n] conditional, y[n:2n] null), v = u + s (c - u);
//   dup != 0 writes v into both halves of v_out [2 n_img, C, H, W] (forward_with_cfg returns cat[v, v]).
//   x_whole: x is the whole input of a conditioned network (see run_unet_program).
static int eval_velocity(lfm_ctx* ctx, cudaStream_t s, const float* t, int t_numel, const float* x, int n_img,
                         const long long* y, float cfg_scale, int dup, float* v_out, bool x_whole = false) {
    const size_t n = (size_t)n_img * ctx->out_chw;
    if (cfg_scale > 1.0f && ctx->net == NetKind::ADM)
        return fail(ctx, "UNetModel has no forward_with_cfg (reference models/guided_diffusion/unet.py): cfg_scale must be <= 1");
    if (cfg_scale > 1.0f) {
        if (launch_network(ctx, s, t, t_numel, x, n_img, y, 2 * n_img, x_whole)) return 1;
        cfg_combine_kernel<<<blocks_for(n), 256, 0, s>>>(ctx->v_net, v_out, n, cfg_scale, dup);
        LAUNCH_OK();
    } else {
        if (launch_network(ctx, s, t, t_numel, x, n_img, y, n_img, x_whole)) return 1;
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

// check_ready for the entries that evaluate the velocity network (lfm_forward, lfm_sample_*), which a VAE context has not.
static int check_velocity_ready(lfm_ctx* ctx, int rows, const char* who) {
    if (check_ready(ctx, rows, who)) return 1;
    if (ctx->net == NetKind::VAE || ctx->net == NetKind::VAE_ENC)
        return fail(ctx, "%s: a VAE context (lfm_create_vae / lfm_create_vae_encoder) has no velocity network", who);
    return 0;
}

// A concat-conditioned context (in_channels > out_channels) evaluates its network on [state | stored condition]: the samplers run
// only with a condition for exactly their B_img images.
static int check_condition(lfm_ctx* ctx, int B_img, const char* who) {
    const UNetState* u = ctx->un;
    if (u == nullptr || u->cond_ch == 0 || u->cond_rows == B_img) return 0;
    return fail(ctx, "%s: the context is concat-conditioned (%d condition channels): call lfm_set_condition for exactly %d images "
                     "first (the stored condition holds %d)", who, u->cond_ch, B_img, u->cond_rows);
}

extern "C" int lfm_forward(lfm_ctx* ctx, const float* t, int t_numel, const float* x, const int64_t* y, int B,
                           float cfg_scale, float* v_out, void* stream) {
    if (check_velocity_ready(ctx, B, "lfm_forward")) return 1;
    if (t == nullptr || x == nullptr || v_out == nullptr) return fail(ctx, "lfm_forward: null tensor");
    if (t_numel != 1 && t_numel != B) return fail(ctx, "lfm_forward: t has %d elements, expected 1 or %d", t_numel, B);
    if (bind(ctx)) return 1;
    const bool cfg = cfg_scale > 1.0f;
    if (cfg && B % 2 != 0) return fail(ctx, "lfm_forward: forward_with_cfg needs an even batch (got %d)", B);
    // a conditioned context takes x as the whole network input [B, in_channels, H, W] (WrapperCondFlow's cat([x, cond], 1))
    const bool x_whole = ctx->un != nullptr && ctx->un->cond_ch > 0;
    // under CFG a vector t has 2n entries in the reference; both halves carry the same times (the x halves are identical)
    return eval_velocity(ctx, static_cast<cudaStream_t>(stream), t, t_numel, x, cfg ? B / 2 : B,
                         reinterpret_cast<const long long*>(y), cfg_scale, 1, v_out, x_whole);
}

extern "C" int lfm_set_condition(lfm_ctx* ctx, const float* cond, int B_img, int channels, void* stream) {
    if (ctx == nullptr) return fail(ctx, "lfm_set_condition: null ctx");
    if (ctx->net != NetKind::ADM || ctx->un->cond_ch == 0)
        return fail(ctx, "lfm_set_condition: the context is not concat-conditioned (lfm_create_unet with in_channels > out_channels)");
    UNetState* u = ctx->un;
    if (channels != u->cond_ch)
        return fail(ctx, "lfm_set_condition: channels must be in_channels - out_channels = %d (got %d)", u->cond_ch, channels);
    if (!ctx->finalized) return fail(ctx, "lfm_set_condition: lfm_finalize has not been called");
    if (B_img < 1 || B_img > ctx->max_rows)
        return fail(ctx, "lfm_set_condition: B_img must be in [1, %d], the finalized rows (got %d)", ctx->max_rows, B_img);
    if (cond == nullptr) return fail(ctx, "lfm_set_condition: cond must not be NULL");
    if (bind(ctx)) return 1;
    CUDA_OK(cudaMemcpyAsync(u->cond, cond, (size_t)B_img * channels * u->S * u->S * sizeof(float), cudaMemcpyDeviceToDevice,
                            static_cast<cudaStream_t>(stream)));
    u->cond_rows = B_img;
    return 0;
}

// ------------------------------------------------------------------------------------------------
// step graphs: each step of a fixed-step solver and each attempted step of an adaptive one is one captured graph,
// replayed from the host

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

// The graph cached under `key`, or a new one: `record` enqueues one step into ctx->stream.  A warm-up run outside of
// capture sets the lazily set function attributes and counts the kernels of one replay; a second run is captured.
// The warm-up runs on the live solver state, so callers initialise that state after this call.
template <typename Record>
static int get_graph(lfm_ctx* ctx, const char* key, Record&& record, lfm_ctx::StepGraph* out) {
    auto it = ctx->graphs.find(key);
    if (it != ctx->graphs.end()) {
        *out = it->second;
        return 0;
    }
    const int64_t launches_before = ctx->launches;
    if (record()) return 1;
    CUDA_OK(cudaStreamSynchronize(ctx->stream));
    lfm_ctx::StepGraph g;
    g.launches = static_cast<int>(ctx->launches - launches_before);
    cudaGraph_t graph = nullptr;
    CUDA_OK(cudaStreamBeginCapture(ctx->stream, cudaStreamCaptureModeThreadLocal));
    const int rc = record();
    cudaError_t e = cudaStreamEndCapture(ctx->stream, &graph);
    ctx->launches = launches_before;
    if (rc) return 1;
    if (e != cudaSuccess) return fail(ctx, "graph capture failed: %s", cudaGetErrorString(e));
    CUDA_OK(cudaGraphInstantiate(&g.exec, graph, 0));
    CUDA_OK(cudaGraphDestroy(graph));
    ctx->graphs[key] = g;
    *out = g;
    return 0;
}

// ------------------------------------------------------------------------------------------------
// fixed-step solvers

// One interval of `method` (LFM_METHOD_*), recorded into ctx->stream.  The interval index is the device counter
// ctx->step_state: the step copies its S stage times from ctx->t_stage into t_eval[0..S), evaluates the network at
// t_eval + j into k[j], and the update kernels read dt from the nodes ctx->t_grid.
static int record_fixed_step(lfm_ctx* ctx, int method, int S, int n_img, bool has_y, float cfg_scale) {
    cudaStream_t s = ctx->stream;
    const size_t n = (size_t)n_img * ctx->out_chw;
    const long long* y = has_y ? ctx->y_buf : nullptr;
    const float* tg = ctx->t_grid;
    const StepState* st = ctx->step_state;
    float* x = ctx->x_state;
    float* xs = ctx->x_pred;  // input of the later stages
    float** k = ctx->kbuf;
    stage_time_kernel<<<1, 32, 0, s>>>(ctx->t_stage, st, S, ctx->t_eval);
    LAUNCH_OK();
    auto eval = [&](int j, const float* xin) {
        return eval_velocity(ctx, s, ctx->t_eval + j, 1, xin, n_img, y, cfg_scale, 0, k[j]);
    };
    auto stage = [&](int mode, float* out) {
        fixed_rk_stage_kernel<<<blocks_for(n), 256, 0, s>>>(mode, x, k[0], k[1], k[2], k[3], tg, st, out, n);
        LAUNCH_OK();
        return 0;
    };
    if (method == LFM_METHOD_EULER) {
        if (eval(0, x)) return 1;
        euler_update_kernel<<<blocks_for(n), 256, 0, s>>>(x, k[0], tg, st, n);
        LAUNCH_OK();
    } else if (method == LFM_METHOD_HEUN) {
        if (eval(0, x)) return 1;
        heun_predict_kernel<<<blocks_for(n), 256, 0, s>>>(x, k[0], xs, tg, st, n);
        LAUNCH_OK();
        if (eval(1, xs)) return 1;
        heun_correct_kernel<<<blocks_for(n), 256, 0, s>>>(x, k[0], k[1], tg, st, n);
        LAUNCH_OK();
    } else if (method == LFM_METHOD_MIDPOINT) {
        if (eval(0, x) || stage(0, xs) || eval(1, xs) || stage(1, x)) return 1;
    } else {
        if (eval(0, x) || stage(2, xs) || eval(1, xs) || stage(3, xs) || eval(2, xs) || stage(4, xs) || eval(3, xs) ||
            stage(5, x))
            return 1;
    }
    step_advance_kernel<<<1, 32, 0, s>>>(ctx->step_state);
    LAUNCH_OK();
    return 0;
}

extern "C" int lfm_sample_fixed(lfm_ctx* ctx, int method, float* x_inout, const float* t_grid_host, int n_grid,
                                int t_as_vector, int heun_corrector_limit, const int64_t* y, int B_img, float cfg_scale,
                                lfm_ode_stats* stats, void* stream) {
    // bit 0 (t as a [B] vector): a vector of equal times and a 0-d time give the same conditioning vector - nothing to do
    const int perturb = (t_as_vector & LFM_FIXED_PERTURB) ? 1 : 0;
    if (perturb && method == LFM_METHOD_HEUN) return fail(ctx, "lfm_sample_fixed: perturb applies to the torchdiffeq grids (euler, midpoint, rk4)");
    const int rows = cfg_scale > 1.0f ? 2 * B_img : B_img;
    if (check_velocity_ready(ctx, rows, "lfm_sample_fixed") || check_condition(ctx, B_img, "lfm_sample_fixed")) return 1;
    if (method < LFM_METHOD_EULER || method > LFM_METHOD_RK4) return fail(ctx, "lfm_sample_fixed: unknown method %d", method);
    if (n_grid < 2 || n_grid > 8192) return fail(ctx, "lfm_sample_fixed: n_grid must be in [2, 8192] (got %d)", n_grid);
    if (x_inout == nullptr || t_grid_host == nullptr) return fail(ctx, "lfm_sample_fixed: null tensor");
    if (cfg_scale > 1.0f && y == nullptr) return fail(ctx, "lfm_sample_fixed: CFG needs labels");
    const int n_int = n_grid - 1, S = method == LFM_METHOD_EULER ? 1 : method == LFM_METHOD_RK4 ? 4 : 2;
    if (method >= LFM_METHOD_MIDPOINT && n_int * S > 8192) return fail(ctx, "lfm_sample_fixed: too many stages (%d)", n_int * S);
    if (bind(ctx)) return 1;
    cudaStream_t user = static_cast<cudaStream_t>(stream);
    const size_t n = (size_t)B_img * ctx->out_chw;
    const bool has_y = y != nullptr;
    if (join_in(ctx, user)) return 1;
    cudaStream_t s = ctx->stream;

    // The stage times of the whole trajectory, computed here in fp32 exactly as the Python expressions do
    // (t0 + dt * (1/3) ...).  options["perturb"]: the first evaluation of a step one ulp past t0 (Perturb.NEXT), rk4's
    // last one ulp before t1 (Perturb.PREV) - in torchdiffeq's negated time; here in model time the directions flip.
    std::vector<float> tg(n_grid), ts((size_t)n_int * S);
    cudaPointerAttributes pa{};
    CUDA_OK(cudaPointerGetAttributes(&pa, t_grid_host));
    if (pa.type == cudaMemoryTypeDevice || pa.type == cudaMemoryTypeManaged)
        CUDA_OK(cudaMemcpy(tg.data(), t_grid_host, n_grid * sizeof(float), cudaMemcpyDeviceToHost));
    else  // a host array is read directly: cudaMemcpy between two pageable buffers is a driver-staged copy
        memcpy(tg.data(), t_grid_host, n_grid * sizeof(float));
    const float third = (float)(1.0 / 3.0), two_thirds = (float)(2.0 / 3.0);
    for (int i = 0; i < n_int; ++i) {
        const float t0 = tg[i], t1 = tg[i + 1], dt = t1 - t0;
        float* ti = &ts[(size_t)i * S];
        ti[0] = perturb ? nextafterf(t0, t0 - 1.0f) : t0;
        if (method == LFM_METHOD_HEUN) {
            ti[1] = t1;
        } else if (method == LFM_METHOD_MIDPOINT) {
            ti[1] = t0 + 0.5f * dt;
        } else if (method == LFM_METHOD_RK4) {
            ti[1] = t0 + dt * third;
            ti[2] = t0 + dt * two_thirds;
            ti[3] = perturb ? nextafterf(t1, t1 + 1.0f) : t1;
        }
    }
    CUDA_OK(cudaMemcpyAsync(ctx->t_grid, tg.data(), tg.size() * sizeof(float), cudaMemcpyHostToDevice, s));
    CUDA_OK(cudaMemcpyAsync(ctx->t_stage, ts.data(), ts.size() * sizeof(float), cudaMemcpyHostToDevice, s));
    if (has_y) CUDA_OK(cudaMemcpyAsync(ctx->y_buf, y, (size_t)rows * sizeof(long long), cudaMemcpyDefault, s));

    // The step graphs.  Heun's intervals past the corrector limit replay an Euler step on stage 0 of the Heun table.
    // A new graph's warm-up run reads the step counter (reset first: the table index scales with S) and clobbers
    // the counter and the state, which are initialised afterwards.
    const int n_main = method == LFM_METHOD_HEUN ? std::min(std::max(heun_corrector_limit, 0), n_int) : n_int;
    auto step_graph = [&](int m, lfm_ctx::StepGraph* g) {
        char key[128];
        snprintf(key, sizeof(key), "m%d_s%d_n%d_y%d_c%.6f", m, S, B_img, has_y ? 1 : 0, cfg_scale > 1.0f ? cfg_scale : 0.f);
        return get_graph(ctx, key, [&] { return record_fixed_step(ctx, m, S, B_img, has_y, cfg_scale); }, g);
    };
    lfm_ctx::StepGraph g_main, g_tail;
    CUDA_OK(cudaMemsetAsync(ctx->step_state, 0, sizeof(StepState), s));
    if (n_main > 0 && step_graph(method, &g_main)) return 1;
    if (n_main < n_int && step_graph(LFM_METHOD_EULER, &g_tail)) return 1;
    CUDA_OK(cudaMemsetAsync(ctx->step_state, 0, sizeof(StepState), s));
    CUDA_OK(cudaMemcpyAsync(ctx->x_state, x_inout, n * sizeof(float), cudaMemcpyDeviceToDevice, s));
    CUDA_OK(cudaStreamSynchronize(s));  // tg / ts are pageable host memory
    int64_t nfe = 0;
    for (int i = 0; i < n_int; ++i) {
        const bool main_kind = i < n_main;
        CUDA_OK(cudaGraphLaunch(main_kind ? g_main.exec : g_tail.exec, s));
        ctx->launches += main_kind ? g_main.launches : g_tail.launches;
        nfe += main_kind ? S : 1;
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
};

// k_out = -v(t = -s_time, y)   (model sees a 0-d fp32 time)
static int dp_func(Dopri& d, float s_time, const float* yv, float* k_out) {
    lfm_ctx* ctx = d.ctx;
    const float t = -s_time;
    set_scalar_kernel<<<1, 32, 0, d.s>>>(ctx->t_eval, t);  // by-value launch argument: no host synchronisation
    LAUNCH_OK();
    if (eval_velocity(ctx, d.s, ctx->t_eval, 1, yv, d.n_img, d.y, d.cfg_scale, 0, k_out)) return 1;
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
        if (eval_velocity(ctx, s, ctx->dp_dev->t + i, 1, yi, d.n_img, d.y, d.cfg_scale, 0, ctx->kbuf[i + 1])) return 1;
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

extern "C" int lfm_sample_dopri5(lfm_ctx* ctx, float* x_inout, double t0, double t1, double rtol, double atol,
                                 const int64_t* y, int B_img, float cfg_scale, lfm_ode_stats* stats, void* stream) {
    return lfm_sample_adaptive(ctx, LFM_ADAPTIVE_DOPRI5, x_inout, t0, t1, rtol, atol, y, B_img, cfg_scale, stats, stream);
}

extern "C" int lfm_sample_adaptive(lfm_ctx* ctx, int method, float* x_inout, double t0, double t1, double rtol, double atol,
                                   const int64_t* y, int B_img, float cfg_scale, lfm_ode_stats* stats, void* stream) {
    const int rows = cfg_scale > 1.0f ? 2 * B_img : B_img;
    if (check_velocity_ready(ctx, rows, "lfm_sample_adaptive") || check_condition(ctx, B_img, "lfm_sample_adaptive")) return 1;
    if (method < LFM_ADAPTIVE_DOPRI5 || method > LFM_ADAPTIVE_HEUN) return fail(ctx, "lfm_sample_adaptive: unknown method %d", method);
    if (x_inout == nullptr) return fail(ctx, "lfm_sample_adaptive: null tensor");
    if (!(t0 > t1)) return fail(ctx, "lfm_sample_adaptive: expects t0 > t1 (reference integrates t: 1 -> 0)");
    if (cfg_scale > 1.0f && y == nullptr) return fail(ctx, "lfm_sample_adaptive: CFG needs labels");
    if (bind(ctx)) return 1;
    cudaStream_t user = static_cast<cudaStream_t>(stream);
    if (join_in(ctx, user)) return 1;
    Dopri d{ctx, ctx->stream, B_img, nullptr, cfg_scale, (size_t)B_img * ctx->out_chw};
    d.tab = make_tableau(method);
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

    // the step graph first: its warm-up run scribbles over the scratch buffers ytmp, y1, k2..k7 and ratio (never over
    // y0 / k1, set below)
    lfm_ctx::StepGraph g_step;
    CUDA_OK(cudaMemsetAsync(ctx->dp_dev, 0, sizeof(DpStep), s));
    char key[160];
    snprintf(key, sizeof(key), "dp%d_n%d_y%d_c%.6f_a%.9g_r%.9g", method, B_img, d.y != nullptr ? 1 : 0,
             cfg_scale > 1.0f ? cfg_scale : 0.f, atol_f, rtol_f);
    if (get_graph(ctx, key, [&] { return dp_record_step(d, atol_f, rtol_f); }, &g_step)) return 1;

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
        CUDA_OK(cudaGraphLaunch(g_step.exec, s));
        ctx->launches += g_step.launches;
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

// Runs one kernel-level entry's launches, `op(ctx)`, on the current device, after its arguments are checked.  `ctx` stands in
// for the network context: it receives the error message and counts the launches.  lfm_label_condition, which needs no
// context either, runs through it too.
template <typename Op>
static int dbg_run(Op&& op) {
    g_num_sms = query_num_sms();
    if (g_num_sms <= 0) return fail(nullptr, "no CUDA device");
    lfm_ctx dbg;
    return op(&dbg);
}

// The GEMM entries' body: lfm_dbg_gemm, _reversed and _path on bf16 operands, lfm_dbg_gemm_fp8 (Op = __nv_fp8_e4m3) on e4m3 ones with
// their row scales a_scale and w_scale.  `reverse` sets GemmEpi::reverse_m, as the network does on every other GEMM.  tma_store = 0 / 1
// forces the epilogue's stores.  By default (-1) the output is stored through a tensor map whenever one can be made for it (16-byte
// aligned base and pitch), as in the network.
template <typename Op = __nv_bfloat16>
static int dbg_gemm(const char* who, int reverse, const void* a, const void* w, const float* bias, void* out, const float* gate,
                    int gate_stride, int rows_per_sample, int M, int N, int K, int epi, int block_n, void* stream, int tma_store = -1,
                    const float* a_scale = nullptr, const float* w_scale = nullptr) {
    constexpr bool e4m3 = std::is_same_v<Op, __nv_fp8_e4m3>;
    if (M < 1 || N < 8 || N % 8 != 0 || K < 1 || K % gemm_block_k<Op>() != 0)
        return fail(nullptr, "%s: K, M or N out of range: M must be >= 1, N a positive multiple of 8 and K of %d (got M %d, N %d, K %d)",
                    who, gemm_block_k<Op>(), M, N, K);
    if (e4m3 && epi != EPI_BIAS_BF16 && epi != EPI_BIAS_GELU_BF16)
        return fail(nullptr, "%s: epi must be 0 (bias -> bf16) or 1 (bias + GELU -> bf16) (got %d)", who, epi);
    if (epi < EPI_BIAS_BF16 || epi > EPI_BIAS_F32) return fail(nullptr, "%s: unknown epilogue %d", who, epi);
    if (block_n != 0 && block_n != 128 && block_n != 256)
        return fail(nullptr, "%s: block_n must be 0, 128 or 256 (got %d)", who, block_n);
    if (tma_store < -1 || tma_store > 1) return fail(nullptr, "%s: tma_store must be -1, 0 or 1 (got %d)", who, tma_store);
    if (e4m3 && (a == nullptr || a_scale == nullptr || w == nullptr || w_scale == nullptr || out == nullptr))
        return fail(nullptr, "%s: a, a_scale, w, w_scale and out must not be NULL (bias may be)", who);
    return dbg_run([&](lfm_ctx* ctx) {
        CUtensorMap ta, tb, tc;
        if (!make_tmap_operand<Op>(&ta, a, M, K) || !make_tmap_operand<Op>(&tb, w, N, K))
            return fail(ctx, "%s: tensor map encode failed", who);
        const bool has_c = tma_store != 0 && make_tmap_out(&tc, out, M, N, N, epi >= EPI_GATE_RESID_F32);
        if (tma_store == 1 && !has_c) return fail(ctx, "%s: no output tensor map for this output (16-byte alignment)", who);
        GemmEpi ep{bias, out, N, gate, gate_stride, rows_per_sample > 0 ? rows_per_sample : 1};
        ep.reverse_m = reverse;
        ep.out_map = has_c ? &tc : nullptr;
        ep.a_scale = a_scale;
        ep.w_scale = w_scale;
        CUDA_OK(launch_gemm<Op>(static_cast<cudaStream_t>(stream), ta, tb, M, N, K, epi, block_n, ep));
        return 0;
    });
}

extern "C" int lfm_dbg_gemm(const void* a_bf16, const void* w_bf16, const float* bias, void* out, const float* gate,
                            int gate_stride, int rows_per_sample, int M, int N, int K, int epi, int block_n,
                            void* stream) {
    return dbg_gemm("lfm_dbg_gemm", 0, a_bf16, w_bf16, bias, out, gate, gate_stride, rows_per_sample, M, N, K, epi, block_n, stream);
}

extern "C" int lfm_dbg_gemm_reversed(const void* a_bf16, const void* w_bf16, const float* bias, void* out, const float* gate,
                                     int gate_stride, int rows_per_sample, int M, int N, int K, int epi, int block_n,
                                     void* stream) {
    return dbg_gemm("lfm_dbg_gemm_reversed", 1, a_bf16, w_bf16, bias, out, gate, gate_stride, rows_per_sample, M, N, K, epi, block_n,
                    stream);
}

extern "C" int lfm_dbg_gemm_path(const void* a_bf16, const void* w_bf16, const float* bias, void* out, const float* gate,
                                 int gate_stride, int rows_per_sample, int M, int N, int K, int epi, int block_n, int reverse,
                                 int tma_store, void* stream) {
    return dbg_gemm("lfm_dbg_gemm_path", reverse != 0, a_bf16, w_bf16, bias, out, gate, gate_stride, rows_per_sample, M, N, K, epi,
                    block_n, stream, tma_store);
}

// The DiT's own kernels, each through the helper launch_network calls.

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// The body of lfm_dbg_ln_modulate (OutT = bf16) and lfm_dbg_ln_modulate_fp8 (e4m3 codes and their row scales ys).
template <typename OutT>
static int dbg_ln_modulate(const char* who, const float* x, void* y, float* ys, const float* shift, const float* scale, int mod_stride,
                           int rows_per_sample, int M, int D, int down, void* stream) {
    constexpr bool e4m3 = std::is_same_v<OutT, __nv_fp8_e4m3>;
    if (!ln_width_ok(D)) return fail(nullptr, "%s: D must be 128 x {2, 3, 6, 8, 9} (got %d)", who, D);
    if (!ln_rows_per_sample_ok(rows_per_sample))
        return fail(nullptr, "%s: rows_per_sample must be a positive multiple of %d (got %d)", who, kLnRows, rows_per_sample);
    if (M < 1) return fail(nullptr, "%s: M must be >= 1 (got %d)", who, M);
    if (mod_stride < 0 || mod_stride % 4 != 0)
        return fail(nullptr, "%s: mod_stride must be a non-negative multiple of 4 (got %d)", who, mod_stride);
    if (down != 0 && down != 1) return fail(nullptr, "%s: down must be 0 or 1 (got %d)", who, down);
    if (x == nullptr || y == nullptr || shift == nullptr || scale == nullptr || (e4m3 && ys == nullptr))
        return fail(nullptr, "%s: x, y, %sshift and scale must not be NULL", who, e4m3 ? "y_scale, " : "");
    if (!aligned16(x) || !aligned16(y) || !aligned16(shift) || !aligned16(scale))
        return fail(nullptr, "%s: x, y, shift and scale must be 16-byte aligned", who);
    return dbg_run([&](lfm_ctx* ctx) {
        COUNT_LAUNCH(launch_ln(static_cast<cudaStream_t>(stream), x, static_cast<OutT*>(y), shift, scale, mod_stride, rows_per_sample, M,
                               D, down, ys));
        return 0;
    });
}

extern "C" int lfm_dbg_ln_modulate(const float* x, void* y_bf16, const float* shift, const float* scale, int mod_stride,
                                   int rows_per_sample, int M, int D, int down, void* stream) {
    return dbg_ln_modulate<__nv_bfloat16>("lfm_dbg_ln_modulate", x, y_bf16, nullptr, shift, scale, mod_stride, rows_per_sample, M, D,
                                          down, stream);
}

// The FP8 mode's kernels, through the launch helpers the DiT forward and lfm_set_param use.

extern "C" int lfm_dbg_gemm_fp8(const void* a_e4m3, const float* a_scale, const void* w_e4m3, const float* w_scale, const float* bias,
                                void* out_bf16, int M, int N, int K, int epi, int block_n, void* stream) {
    return dbg_gemm<__nv_fp8_e4m3>("lfm_dbg_gemm_fp8", 0, a_e4m3, w_e4m3, bias, out_bf16, nullptr, 0, 1, M, N, K, epi, block_n, stream, -1,
                                   a_scale, w_scale);
}

extern "C" int lfm_dbg_ln_modulate_fp8(const float* x, void* y_e4m3, float* y_scale, const float* shift, const float* scale, int mod_stride,
                                       int rows_per_sample, int M, int D, int down, void* stream) {
    return dbg_ln_modulate<__nv_fp8_e4m3>("lfm_dbg_ln_modulate_fp8", x, y_e4m3, y_scale, shift, scale, mod_stride, rows_per_sample, M, D,
                                          down, stream);
}

extern "C" int lfm_dbg_quantize_rows_fp8(const float* w, void* codes_e4m3, float* scales, int N, int K, void* stream) {
    if (N < 1 || K < 1) return fail(nullptr, "lfm_dbg_quantize_rows_fp8: N and K must be >= 1 (got N %d, K %d)", N, K);
    if (w == nullptr || codes_e4m3 == nullptr || scales == nullptr)
        return fail(nullptr, "lfm_dbg_quantize_rows_fp8: w, codes and scales must not be NULL");
    return dbg_run([&](lfm_ctx* ctx) {
        launch_quantize_rows_e4m3(static_cast<cudaStream_t>(stream), w, static_cast<__nv_fp8_e4m3*>(codes_e4m3), scales, N, K);
        LAUNCH_OK();
        return 0;
    });
}

extern "C" int lfm_dbg_condition(const float* t, int t_numel, const long long* y, int rows, int feat, int E, const float* w0,
                                 const float* b0, const float* w2, const float* b2, const float* table, int max_row, int null_row,
                                 float* tf_out, float* h1_out, void* c_bf16, void* stream) {
    if (rows < 1) return fail(nullptr, "lfm_dbg_condition: rows must be >= 1 (got %d)", rows);
    if (t_numel != 1 && t_numel != rows)
        return fail(nullptr, "lfm_dbg_condition: t_numel must be 1 or rows (got %d, rows %d)", t_numel, rows);
    if (!condition_k_ok(feat) || !condition_k_ok(E))
        return fail(nullptr, "lfm_dbg_condition: feat and E must be multiples of 128 up to %d (got feat %d, E %d)", kConditionMaxK, feat, E);
    if (max_row < 0 || null_row < -1 || null_row > max_row)
        return fail(nullptr, "lfm_dbg_condition: max_row must be >= 0 and null_row in [-1, max_row] (got %d, %d)", max_row, null_row);
    if (t == nullptr || w0 == nullptr || b0 == nullptr || w2 == nullptr || b2 == nullptr || tf_out == nullptr || h1_out == nullptr ||
        c_bf16 == nullptr || (table == nullptr && (y != nullptr || null_row >= 0)))
        return fail(nullptr, "lfm_dbg_condition: only y may be NULL, and table when neither y nor null_row reads it");
    return dbg_run([&](lfm_ctx* ctx) {
        return launch_condition(ctx, static_cast<cudaStream_t>(stream), t, t_numel, y, rows, feat, E, w0, b0, w2, b2, table, max_row,
                                null_row, tf_out, h1_out, static_cast<__nv_bfloat16*>(c_bf16));
    });
}

extern "C" int lfm_dbg_patch_embed(const float* x, int x_rows, const float* Wt, const float* bias, const float* pos, float* tok, int D,
                                   int G, int C, int p, int M, void* stream) {
    if (!dit_patch_ok(p)) return fail(nullptr, "lfm_dbg_patch_embed: p must be 2, 4 or 8 (got %d)", p);
    if (p == 2 ? C != 4 : (C < 1 || 8 * C * p * p * (int)sizeof(float) > 48 * 1024))
        return fail(nullptr, "lfm_dbg_patch_embed: C must be 4 at p = 2, and 8 C p^2 floats must fit 48 KB (got C %d, p %d)", C, p);
    if (D < 4 || D % 4 != 0) return fail(nullptr, "lfm_dbg_patch_embed: D must be a positive multiple of 4 (got %d)", D);
    if (G < 1 || x_rows < 1 || M < 1)
        return fail(nullptr, "lfm_dbg_patch_embed: G, x_rows and M must be >= 1 (got %d, %d, %d)", G, x_rows, M);
    if (x == nullptr || Wt == nullptr || bias == nullptr || pos == nullptr || tok == nullptr)
        return fail(nullptr, "lfm_dbg_patch_embed: x, Wt, bias, pos and tok must not be NULL");
    return dbg_run([&](lfm_ctx* ctx) {
        return launch_patch_embed(ctx, static_cast<cudaStream_t>(stream), x, x_rows, Wt, bias, pos, tok, D, G, C, p, M);
    });
}

extern "C" int lfm_dbg_final_layer(const float* x, const float* shift, const float* scale, int mod_stride, const float* W, const float* bias,
                                   float* v_net, int M, int D, int G, int C, int p, void* stream) {
    if (!dit_patch_ok(p)) return fail(nullptr, "lfm_dbg_final_layer: p must be 2, 4 or 8 (got %d)", p);
    if (p == 2 ? C != 4 : C < 1)
        return fail(nullptr, "lfm_dbg_final_layer: C must be 4 at p = 2 (the kernel computes 16 outputs), >= 1 otherwise (got %d)", C);
    if (D < 128 || D % 128 != 0 || D > kFinalLayerMaxD)
        return fail(nullptr, "lfm_dbg_final_layer: D must be a multiple of 128 up to %d (got %d)", kFinalLayerMaxD, D);
    if (mod_stride < 0 || mod_stride % 4 != 0)
        return fail(nullptr, "lfm_dbg_final_layer: mod_stride must be a non-negative multiple of 4 (got %d)", mod_stride);
    if (G < 1 || M < 1) return fail(nullptr, "lfm_dbg_final_layer: G and M must be >= 1 (got %d, %d)", G, M);
    if (x == nullptr || shift == nullptr || scale == nullptr || W == nullptr || bias == nullptr || v_net == nullptr ||
        !aligned16(shift) || !aligned16(scale))
        return fail(nullptr, "lfm_dbg_final_layer: x, shift, scale, W, bias and v_net must not be NULL (shift and scale 16-byte aligned)");
    return dbg_run([&](lfm_ctx* ctx) {
        return launch_final_layer(ctx, static_cast<cudaStream_t>(stream), x, shift, scale, mod_stride, W, bias, v_net, M, D, G, C, p);
    });
}

extern "C" int lfm_dbg_attention(const void* qkv_bf16, void* out_bf16, int B, int T, int heads, int ch, int head_dim, int layout,
                                 void* stream) {
    if (layout != LFM_QKV_TIMM && layout != LFM_QKV_HEAD_MAJOR)
        return fail(nullptr, "lfm_dbg_attention: layout must be LFM_QKV_TIMM (0) or LFM_QKV_HEAD_MAJOR (1) (got %d)", layout);
    if (B < 1 || heads < 1) return fail(nullptr, "lfm_dbg_attention: B and heads must be >= 1 (got B %d, heads %d)", B, heads);
    if (head_dim < 1 || head_dim > ch) return fail(nullptr, "lfm_dbg_attention: head_dim must be in [1, ch] (got head_dim %d, ch %d)", head_dim, ch);
    const AttnKernel k = attn_route(T, ch, layout);
    if (k == AttnKernel::NONE)
        return fail(nullptr, "lfm_dbg_attention: %d tokens with a head width of %d channels in the %s layout are not supported", T, ch,
                    layout == LFM_QKV_TIMM ? "timm" : "head-major");
    if (head_dim < ch && !attn_takes_padded_heads(k))
        return fail(nullptr, "lfm_dbg_attention: head_dim %d < ch: the kernel for %d tokens with %d channels takes no padded heads", head_dim,
                    T, ch);
    if (qkv_bf16 == nullptr || out_bf16 == nullptr) return fail(nullptr, "lfm_dbg_attention: qkv and out must not be NULL");
    return dbg_run([&](lfm_ctx* ctx) {
        AttnOp op;
        if (!attn_plan(&op, static_cast<const __nv_bfloat16*>(qkv_bf16), static_cast<__nv_bfloat16*>(out_bf16), T, ch, head_dim, heads,
                       layout, B))
            return fail(ctx, "lfm_dbg_attention: tensor map encode failed");
        CUDA_OK(launch_attention(op, static_cast<cudaStream_t>(stream), B));
        return 0;
    });
}

// The entries below run one op of the UNet program through the program's own construction (push_*) and launch (run_*_op) helpers.

static bool conv_out_side_ok(int s) { return s == 4 || s == 8 || s == 16 || s == 32 || s == 64 || s == 128 || s == 256; }

// lfm_dbg_conv, lfm_dbg_conv_wide and lfm_dbg_conv_down: the argument checks, then the launch.  The mode selects the geometry
// and split-K rule: CONV, lfm_dbg_conv's (output side 4..256, stride 1 or 2, tap origin 1, ksplit -1 = push_conv's plan, 1 = none,
// or 2..8); WIDE, lfm_dbg_conv_wide's (output side 256 or 512, stride 1, never split along K); DOWN, lfm_dbg_conv_down's (the VAE
// encoder's Downsample2D: stride 2 with tap origin 0, output side 4..256, split-K as CONV).
enum class DbgConv { CONV, WIDE, DOWN };
static int dbg_conv(const char* who, DbgConv mode, const void* x_bf16, const void* w_bf16, const float* bias, void* out,
                    unsigned long long* gn_bins, int B, int side, int Cin, int Cout, int stride, int block_n, int epi, int ksplit,
                    void* stream) {
    const bool wide = mode == DbgConv::WIDE;
    if (mode == DbgConv::DOWN) {
        if (stride != 2) return fail(nullptr, "%s: stride must be 2 (got %d)", who, stride);
        if (side % 2 != 0 || !conv_out_side_ok(side / 2))
            return fail(nullptr, "%s: side must be 8, 16, 32, 64, 128, 256 or 512 (got %d)", who, side);
        if (B < 1 || (long long)B * (side / 2) * (side / 2) > INT32_MAX)
            return fail(nullptr, "%s: B must be >= 1 and B * (side / 2)^2 below 2^31 output pixels (got B %d)", who, B);
    } else if (wide) {
        if (side != 256 && side != 512) return fail(nullptr, "%s: side must be 256 or 512 (got %d)", who, side);
        if (stride != 1) return fail(nullptr, "%s: stride must be 1 (got %d)", who, stride);
        if (B < 1 || (long long)B * side * side > INT32_MAX)
            return fail(nullptr, "%s: B must be >= 1 and B * side^2 below 2^31 output pixels (got B %d)", who, B);
    } else {
        if (B < 1) return fail(nullptr, "%s: B must be >= 1 (got %d)", who, B);
        if (stride != 1 && stride != 2) return fail(nullptr, "%s: stride must be 1 or 2 (got %d)", who, stride);
        if (side % stride != 0 || !conv_out_side_ok(side / stride))
            return fail(nullptr, "%s: side %d with stride %d: the output side must be 4, 8, 16, 32, 64, 128 or 256", who, side, stride);
    }
    if (Cin < 64 || Cin % 64 != 0) return fail(nullptr, "%s: Cin must be a positive multiple of 64 (got %d)", who, Cin);
    if (!(Cout == 4 || (Cout >= 8 && Cout % 8 == 0))) return fail(nullptr, "%s: Cout must be 4 or a multiple of 8 (got %d)", who, Cout);
    if (block_n != 0 && block_n != 128 && block_n != 256) return fail(nullptr, "%s: block_n must be 0, 128 or 256 (got %d)", who, block_n);
    if (epi != EPI_BIAS_F32 && epi != EPI_BIAS_BF16 && epi != EPI_GATE_RESID_F32)
        return fail(nullptr, "%s: epi must be 3 (fp32 out), 0 (bf16 out) or 2 (out += conv) (got %d)", who, epi);
    if (wide) {
        if (ksplit != 1) return fail(nullptr, "%s: ksplit must be 1: wide rows are never split along K (got %d)", who, ksplit);
    } else {
        if (ksplit != -1 && (ksplit < 1 || ksplit > 8))
            return fail(nullptr, "%s: ksplit must be -1 (the network's plan), 1 (none) or 2..8 (got %d)", who, ksplit);
        if (ksplit > 1 && (epi == EPI_BIAS_BF16 || block_n == 256))
            return fail(nullptr, "%s: ksplit %d: split-K writes fp32 (epi 3 or 2) with 128-wide tiles (block_n 0 or 128)", who, ksplit);
    }
    const int out_hw = (side / stride) * (side / stride), cpg = Cout / 32;
    if (gn_bins != nullptr && (epi == EPI_GATE_RESID_F32 || ksplit > 1 || Cout % 32 != 0 ||
                               !(cpg == 4 || cpg == 8 || cpg == 16 || cpg == 32 || cpg == 64) || out_hw % 32 != 0))
        return fail(nullptr, "%s: gn_bins needs epi 3 or 0, no split-K, Cout / 32 in {4, 8, 16, 32, 64} and a multiple of 32 "
                             "output pixels (got epi %d, ksplit %d, Cout %d, %d pixels)", who, epi, ksplit, Cout, out_hw);
    if (x_bf16 == nullptr || w_bf16 == nullptr || bias == nullptr || out == nullptr)
        return fail(nullptr, "%s: x, w, bias and out must not be NULL", who);
    return dbg_run([&](lfm_ctx* ctx) {
        UNetState u;
        if (!push_conv(&u, B, static_cast<const __nv_bfloat16*>(x_bf16), side, Cin, stride, static_cast<const __nv_bfloat16*>(w_bf16),
                       bias, Cout, out, epi, mode == DbgConv::DOWN ? 0 : 1))
            return fail(ctx, "%s: tensor map encode failed", who);
        UOp& o = u.prog[0];
        if (ksplit >= 1) {
            o.ksplit = ksplit;
            o.split_pitch = ksplit > 1 ? (B * out_hw + kGemmBlockM - 1) / kGemmBlockM * kGemmBlockM : 0;
        }
        if (o.ksplit > 1 && (block_n == 256 || gn_bins != nullptr))
            return fail(ctx, "%s: the network splits K %d ways here: pass ksplit 1 for block_n 256 or gn_bins", who, o.ksplit);
        if (gn_bins != nullptr) {
            o.bins_slot = 0;
            u.BINS = gn_bins;
            u.bins_rows = B;
        }
        cudaStream_t s = static_cast<cudaStream_t>(stream);
        if (o.ksplit > 1) CUDA_OK(cudaMallocAsync(&u.SPLIT, (size_t)o.ksplit * o.split_pitch * o.N * sizeof(float), s));
        const int rc = run_gemm_op(ctx, &u, o, s, B, block_n);
        if (u.SPLIT != nullptr) CUDA_OK(cudaFreeAsync(u.SPLIT, s));
        return rc;
    });
}

extern "C" int lfm_dbg_conv(const void* x_bf16, const void* w_bf16, const float* bias, void* out, unsigned long long* gn_bins, int B,
                            int side, int Cin, int Cout, int stride, int block_n, int epi, int ksplit, void* stream) {
    return dbg_conv("lfm_dbg_conv", DbgConv::CONV, x_bf16, w_bf16, bias, out, gn_bins, B, side, Cin, Cout, stride, block_n, epi, ksplit, stream);
}

// Stride-1 3x3 convolutions whose output rows are wider than one 128-pixel tile (the row-segment tiles of the VAE decoder's
// last stages): the same push_conv / run_gemm_op path, never split along K.
extern "C" int lfm_dbg_conv_wide(const void* x_bf16, const void* w_bf16, const float* bias, void* out, unsigned long long* gn_bins,
                                 int B, int side, int Cin, int Cout, int stride, int block_n, int epi, int ksplit, void* stream) {
    return dbg_conv("lfm_dbg_conv_wide", DbgConv::WIDE, x_bf16, w_bf16, bias, out, gn_bins, B, side, Cin, Cout, stride, block_n, epi,
                    ksplit, stream);
}

// The VAE encoder's Downsample2D(padding=0): F.pad(x, (0, 1, 0, 1)) then a 3x3 stride-2 convolution, as the network runs it (tap
// origin 0, the extra bottom row and right column read as the tensor map's zero fill; output rows wider than 128 pixels on
// row segments).  Arguments as lfm_dbg_conv, checked before the device is touched.
extern "C" int lfm_dbg_conv_down(const void* x_bf16, const void* w_bf16, const float* bias, void* out, unsigned long long* gn_bins,
                                 int B, int side, int Cin, int Cout, int stride, int block_n, int epi, int ksplit, void* stream) {
    return dbg_conv("lfm_dbg_conv_down", DbgConv::DOWN, x_bf16, w_bf16, bias, out, gn_bins, B, side, Cin, Cout, stride, block_n, epi,
                    ksplit, stream);
}

// The network's conv_in (input_blocks.0 / conv_in) on the channel concatenation [a | b] of two NCHW fp32 sources.
extern "C" int lfm_dbg_conv_in(const float* a, int a_ch, long long a_stride, const float* b, int b_ch, long long b_stride,
                               const float* w, const float* bias, float* out, int B, int side, int Cout, void* stream) {
    if (a_ch < 1 || b_ch < 0 || a_ch + b_ch < 3 || a_ch + b_ch > kConvInMaxChannels)
        return fail(nullptr, "lfm_dbg_conv_in: a_ch >= 1, b_ch >= 0 and a_ch + b_ch in [3, %d] (got %d, %d)", kConvInMaxChannels, a_ch,
                    b_ch);
    // sides up to 256 for the UNets' latents; 512 for the 3-channel image input of the VAE encoder
    const bool side_ok = (side >= 1 && side <= 256) || (side == 512 && a_ch + b_ch == 3);
    if (!side_ok || conv_in_smem_bytes(a_ch + b_ch, side) > 48 * 1024)
        return fail(nullptr, "lfm_dbg_conv_in: side must be in [1, 256], or 512 with 3 channels, with a_ch + b_ch rows of side + 4 "
                             "floats in 48 KB of shared memory (got side %d, %d channels)", side, a_ch + b_ch);
    if (a_stride < (long long)a_ch * side * side || (b_ch > 0 && b_stride < (long long)b_ch * side * side))
        return fail(nullptr, "lfm_dbg_conv_in: a_stride / b_stride must hold a_ch / b_ch channels of side^2 floats (got %lld, %lld)",
                    a_stride, b_stride);
    if (Cout < 1) return fail(nullptr, "lfm_dbg_conv_in: Cout must be >= 1 (got %d)", Cout);
    if (B < 1 || (long long)B * side > INT32_MAX) return fail(nullptr, "lfm_dbg_conv_in: B must be >= 1 with B * side < 2^31 (got %d)", B);
    if (a == nullptr || (b == nullptr) != (b_ch == 0) || w == nullptr || bias == nullptr || out == nullptr)
        return fail(nullptr, "lfm_dbg_conv_in: a, w, bias and out must not be NULL, and b is NULL exactly when b_ch is 0");
    return dbg_run([&](lfm_ctx* ctx) {
        COUNT_LAUNCH(launch_conv_in(static_cast<cudaStream_t>(stream), ConvInSrc{a, a_ch, a_stride}, ConvInSrc{b, b_ch, b_stride}, B, B,
                                    w, bias, out, side, Cout));
        return 0;
    });
}

// The VAE encoder's tail, vae_quant_kernel: quant_conv (8 -> 8) of conv_out's NHWC fp32 [B * HW, 8] output, then mean and the
// clamped logvar, NCHW fp32 [B, 4, HW].
extern "C" int lfm_dbg_vae_quant(const float* in, const float* w, const float* bias, float* mean, float* logvar, int B, int HW,
                                 void* stream) {
    if (B < 1 || HW < 1 || (long long)B * HW > INT32_MAX)
        return fail(nullptr, "lfm_dbg_vae_quant: B and HW must be >= 1 with B * HW < 2^31 (got %d, %d)", B, HW);
    if (in == nullptr || w == nullptr || bias == nullptr || mean == nullptr || logvar == nullptr || !aligned16(in))
        return fail(nullptr, "lfm_dbg_vae_quant: in, w, bias, mean and logvar must not be NULL (in 16-byte aligned)");
    return dbg_run([&](lfm_ctx* ctx) {
        LAUNCH_K(vae_quant_kernel, dim3(blocks_for((size_t)B * HW)), 256, 0, static_cast<cudaStream_t>(stream), in, w, bias, mean, logvar,
                 B, HW);
        return 0;
    });
}

extern "C" int lfm_dbg_gemm_batched(const void* a_bf16, int a_rows, int a_ld, const void* w_bf16, int w_rows, int w_ld, int K, int N,
                                    void* out, const float* bias, int B, int out_hw, int epi, int batch_m, int a_mod, int b_batch_rows,
                                    void* stream) {
    if (K < 64 || K % 64 != 0 || N < 256 || N % 256 != 0)
        return fail(nullptr, "lfm_dbg_gemm_batched: K must be a multiple of 64 and N of 256 (got K %d, N %d)", K, N);
    if (a_rows < 1 || w_rows < 1 || a_ld < K || w_ld < K || a_ld % 8 != 0 || w_ld % 8 != 0)
        return fail(nullptr, "lfm_dbg_gemm_batched: a_ld / w_ld must be >= K and multiples of 8, a_rows / w_rows >= 1 "
                             "(got a %d x ld %d, w %d x ld %d)", a_rows, a_ld, w_rows, w_ld);
    if (batch_m < 128 || batch_m % 128 != 0 || a_mod < 0 || a_mod % 128 != 0 || b_batch_rows < N)
        return fail(nullptr, "lfm_dbg_gemm_batched: batch_m must be a positive multiple of 128, a_mod 0 or a multiple of 128, "
                             "b_batch_rows >= N (got batch_m %d, a_mod %d, b_batch_rows %d)", batch_m, a_mod, b_batch_rows);
    if (B < 1 || out_hw < 1 || ((long long)B * out_hw) % batch_m != 0)
        return fail(nullptr, "lfm_dbg_gemm_batched: B * out_hw must be a positive multiple of batch_m (got %d x %d)", B, out_hw);
    if (epi != EPI_BIAS_F32 && epi != EPI_BIAS_BF16)
        return fail(nullptr, "lfm_dbg_gemm_batched: epi must be 3 (fp32) or 0 (bf16) (got %d)", epi);
    if (a_bf16 == nullptr || w_bf16 == nullptr || out == nullptr)
        return fail(nullptr, "lfm_dbg_gemm_batched: a, w and out must not be NULL");
    return dbg_run([&](lfm_ctx* ctx) {
        UNetState u;
        if (!push_batched(&u, a_bf16, a_rows, a_ld, K, w_bf16, w_rows, w_ld, N, out, out_hw, epi, bias, batch_m, a_mod, b_batch_rows))
            return fail(ctx, "lfm_dbg_gemm_batched: tensor map encode failed");
        return run_gemm_op(ctx, &u, u.prog[0], static_cast<cudaStream_t>(stream), B, 0);
    });
}

extern "C" int lfm_dbg_groupnorm(const float* a, int Ca, const float* b, int Cb, const void* src_bf16, const unsigned long long* bins,
                                 int max_chunks, const float* gamma, const float* beta, const float* film, int film_stride, int act,
                                 float eps, void* out_bf16, float* copy_out, void* raw_out, int B, int HW, void* stream) {
    const int C = Ca + Cb;
    if (Ca < 4 || Ca % 4 != 0 || Cb < 0 || Cb % 4 != 0 || (b == nullptr) != (Cb == 0))
        return fail(nullptr, "lfm_dbg_groupnorm: Ca must be a positive multiple of 4, Cb 0 (b NULL) or a multiple of 4 (got %d, %d)", Ca, Cb);
    if (C % 128 != 0 || C > 128 * kGnMaxJ)
        return fail(nullptr, "lfm_dbg_groupnorm: Ca + Cb must be a multiple of 128 up to %d (got %d)", 128 * kGnMaxJ, C);
    if (B < 1 || B > 65535 || HW < 1) return fail(nullptr, "lfm_dbg_groupnorm: B must be in [1, 65535] and HW >= 1 (got %d, %d)", B, HW);
    if (bins == nullptr && (max_chunks < 1 || max_chunks > 256))
        return fail(nullptr, "lfm_dbg_groupnorm: max_chunks must be in [1, 256] (got %d)", max_chunks);
    if (act != 0 && act != 1) return fail(nullptr, "lfm_dbg_groupnorm: act must be 0 or 1 (SiLU) (got %d)", act);
    if (film_stride < 0 || !(eps > 0.f)) return fail(nullptr, "lfm_dbg_groupnorm: film_stride must be >= 0 and eps > 0");
    if (a == nullptr || gamma == nullptr || beta == nullptr || out_bf16 == nullptr)
        return fail(nullptr, "lfm_dbg_groupnorm: a, gamma, beta and out must not be NULL");
    return dbg_run([&](lfm_ctx* ctx) {
        UNetState u;
        u.gn_eps = eps;
        u.max_chunks = max_chunks;
        push_gn(&u, Src2{a, b, Ca, Cb}, HW, C, gamma, beta, film, act, static_cast<__nv_bfloat16*>(out_bf16), copy_out,
                static_cast<__nv_bfloat16*>(raw_out));
        UOp& st = u.prog[0];
        UOp& ap = u.prog[1];
        ap.gn_src_bf16 = static_cast<const __nv_bfloat16*>(src_bf16);
        cudaStream_t s = static_cast<cudaStream_t>(stream);
        if (bins != nullptr) {  // statistics from a producing convolution's epilogue: [B][kGnBinReplicas][32 groups][sum, sum of squares]
            st.skip = true;
            ap.bins_slot = 0;
            u.BINS = const_cast<unsigned long long*>(bins);
            u.bins_rows = B;
        } else {
            CUDA_OK(cudaMallocAsync(&u.partial, (size_t)B * max_chunks * 64 * sizeof(double), s));
        }
        int rc = 0;
        for (const UOp& o : u.prog)
            if (rc == 0 && !o.skip) rc = run_gn_op(ctx, &u, o, s, B, film_stride);
        if (u.partial != nullptr) CUDA_OK(cudaFreeAsync(u.partial, s));
        return rc;
    });
}

extern "C" int lfm_dbg_tokens(lfm_ctx* ctx, float* out, int B) {
    if (check_ready(ctx, B, "lfm_dbg_tokens")) return 1;
    if (ctx->net != NetKind::DIT) return fail(ctx, "lfm_dbg_tokens: DiT only");
    CUDA_OK(cudaMemcpy(out, ctx->x_tok, (size_t)B * ctx->T * ctx->D * sizeof(float), cudaMemcpyDefault));
    return 0;
}

// ------------------------------------------------------------------------------------------------
// semantic synthesis: the condition of a batch of label maps (label_condition_kernel)

extern "C" int lfm_label_condition(const uint8_t* labels, int B, int H, int W, int num_classes, int n_stages, const float* weight,
                                   int out_ch, float* out, void* stream) {
    if (num_classes < 1 || num_classes > kLabelCondMaxClasses)
        return fail(nullptr, "lfm_label_condition: num_classes must be in [1, %d] (got %d)", kLabelCondMaxClasses, num_classes);
    if (out_ch < 1 || out_ch > kLabelCondMaxOut)
        return fail(nullptr, "lfm_label_condition: out_ch must be in [1, %d] (got %d)", kLabelCondMaxOut, out_ch);
    if (n_stages < 0 || n_stages > kLabelCondMaxStages)
        return fail(nullptr, "lfm_label_condition: n_stages must be in [0, %d] (got %d)", kLabelCondMaxStages, n_stages);
    const int f = 1 << n_stages;
    if (B < 1 || H < 1 || W < 1 || H % f != 0 || W % f != 0 || (long long)B * H * W > INT32_MAX)
        return fail(nullptr, "lfm_label_condition: H and W must be positive multiples of 2^n_stages = %d, with B * H * W < 2^31 "
                             "(got B %d, H %d, W %d)", f, B, H, W);
    if (labels == nullptr || weight == nullptr || out == nullptr)
        return fail(nullptr, "lfm_label_condition: labels, weight and out must not be NULL");
    return dbg_run([&](lfm_ctx* ctx) {
        static DevOnce once;
        CUDA_OK(smem_opt_in(once, label_condition_kernel, label_cond_smem_bytes(kLabelCondMaxClasses, kLabelCondMaxOut)));
        const int Wo = W >> n_stages, segs = (Wo + kLabelCondPix - 1) / kLabelCondPix;
        LAUNCH_K(label_condition_kernel, dim3(B * (H >> n_stages) * segs), 256, label_cond_smem_bytes(num_classes, out_ch),
                 static_cast<cudaStream_t>(stream), labels, weight, out, H, W, num_classes, out_ch, n_stages);
        return 0;
    });
}
