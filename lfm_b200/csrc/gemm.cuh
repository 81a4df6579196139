// lfm_b200 - persistent, warp-specialised Hopper GEMM (TMA + mbarrier + wgmma) for every linear layer and convolution.
//
//   C[M, N] = A[M, K] * W[N, K]^T   (A: activations bf16 row-major; W: nn.Linear weight, bf16, [out, in])
//
// One 128 x BN output tile per CTA and step of a persistent tile loop (BN = 128 or 256).  Both operands are K-major,
// staged by TMA into 128B-swizzled shared memory (64-element K slabs) in a ring of kStages slots.
// Warp groups (384 threads): group 0 = TMA producer (one thread), groups 1 and 2 = consumers: each multiplies its 64 rows
// of the tile with wgmma.m64nBNk16 into registers (fp32) and applies the fused epilogue to them.  Given an output tensor map
// (GemmEpi::out_map) the epilogue stages 64-row sub-tiles in shared memory and writes each with one TMA store
// (epilogue_tma); otherwise it stores straight from the registers.
//
// Fused epilogues (reference ops they replace):
//   EPI_BIAS_BF16       out = bf16(acc + bias)                       attn.qkv       (timm Attention)
//   EPI_BIAS_GELU_BF16  out = bf16(gelu_tanh(acc + bias))            mlp.fc1 + act  (models/DiT.py:122-124)
//   EPI_GATE_RESID_F32  x  += gate[b] * (acc + bias)   (fp32 stream) attn.proj / mlp.fc2 + gated residual
//                                                                    (models/DiT.py:129-130)
//   EPI_BIAS_F32        out = acc + bias (fp32)                      adaLN_modulation Linears in one GEMM, convolutions
//
// FP8 operands (Op = __nv_fp8_e4m3, plain 2-D GEMMs with EPI_BIAS_BF16 / EPI_BIAS_GELU_BF16, the DiT's qkv and fc1 in its FP8
// mode): A and W hold e4m3 codes with one fp32 scale per A row (GemmEpi::a_scale) and per W row (GemmEpi::w_scale).  A K slab
// is still one 128-byte swizzle row, now 128 elements, so the stage bytes, the ring and the descriptors are those of bf16; each
// slab issues four wgmma.m64nBNk32.e4m3 instead of four k16.bf16, and K must be a multiple of 128.  The epilogue starts from
// acc * a_scale[row] * w_scale[col].
#pragma once
#include "common.cuh"

namespace lfm {

enum EpiMode { EPI_BIAS_BF16 = 0, EPI_BIAS_GELU_BF16 = 1, EPI_GATE_RESID_F32 = 2, EPI_BIAS_F32 = 3 };

struct GemmEpi {
    const float* bias;    // [N] or nullptr
    void* out;            // bf16 [M, ldo] / fp32 [M, ldo]; for EPI_GATE_RESID_F32 the residual stream (read+write)
    int ldo;              // row pitch of out, elements
    const float* gate;    // EPI_GATE_RESID_F32: gate[b * gate_stride + n]; nullptr = gate 1 (plain residual add)
    int gate_stride;      // elements between samples in the modulation table
    int rows_per_sample;  // tokens per sample (b = row / rows_per_sample)
    // Optional (EPI_BIAS_F32 / EPI_BIAS_BF16): GroupNorm statistics of the OUTPUT accumulated in the epilogue -
    // bins[((row / gn_hw) * kGnBinReplicas + r) * 64 + 2 g + {0,1}] += {sum, sum of squares} of group g = column / gn_cpg, as
    // fixed point: the sum in units of 2^-28, the sum of squares in units of 2^-20 (integer atomics => the result does not depend
    // on the order of arrival: deterministic).  The signed 64-bit totals hold |sum| < 2^35 and a sum of squares < 2^43 ~ 8.8e12 per
    // (image, group): rms 2896 at the 512-pixel VAE decode's 512 x 512 x 128 stage (2^20 values per group), 5793 at the
    // 256-pixel decode's 256 x 256 x 128 stage (2^18), 16384 at a 64 x 64 x 256 UNet layer.
    // Each add rounds to half a unit, so at rms 1e-2 the sum of squares of the VAE stage (26.2, from 4096 adds per group) is off by
    // at most 2e-3, 7e-5 relative.  r is any of
    // kGnBinReplicas copies (chosen per warp; the consumer adds them up - integers, so still exact), so that the atomics of
    // all CTAs working on one image do not queue on the same few cache lines.  Needs gn_hw % 16 == 0.
    unsigned long long* gn_bins = nullptr;
    int gn_cpg = 0;
    int gn_hw = 1;
    // Walk the M blocks from the last to the first.  Consecutive kernels of a network alternate direction so that
    // each one starts on the rows its producer touched LAST - the part still resident in L2.
    int reverse_m = 0;
    // Tensor map of `out` (make_tmap_out: 64-row boxes of 128 bytes, 128-byte swizzle), or nullptr.  Given, the epilogue stages
    // each 64-row sub-tile in shared memory and writes it with one TMA store (the residual stream is TMA-loaded into the same
    // buffer first).  The launch passes the map itself as a kernel parameter; the kernel only tests this pointer.  Plain
    // GEMMs without GroupNorm statistics only; sub-tiles with rows past M keep the register stores.
    const CUtensorMap* out_map = nullptr;
    // FP8 operands only: the dequantisation scales of the A rows [M] and of the W rows [N].
    const float* a_scale = nullptr;
    const float* w_scale = nullptr;
};
constexpr int kGnBinReplicas = 16;
constexpr double kGnFixScale = 268435456.0;  // 2^28: the sum
constexpr double kGnFixScaleSq = 1048576.0;  // 2^20: the sum of squares

// Implicit-GEMM convolution geometry (taps == 0: plain GEMM, A is a 2-D [M, K] matrix).
// Output pixels are flattened (b, h, w) row-major; a tile's 128 output rows are whole image rows (W * rows == 128),
// whole images (H * W divides 128) or one 128-pixel segment of an image row (W a multiple of 128: the VAE decoder's last
// stages, W = 256 or 512; make_tmap_act4d refuses any other W above 128), so the matching input window of tap (r, s) is ONE
// 4-D box.  A segment's box starts at w0 - 1 and ends at w0 + 128: the columns left of 0 and right of W - 1 are the TMA's
// zero fill (the padding), the ones across an inner seam are the neighbouring segment's pixels.
// Tap (r, s) of output pixel (h, w) reads input (stride * h + r - pad, stride * w + s - pad).  pad 1 is the symmetric padding of
// every 3x3 convolution but one; pad 0 is diffusers' Downsample2D(padding=0), F.pad(x, (0, 1, 0, 1)) then a stride-2 conv: its
// extra bottom row and right column are the out-of-bounds fill, so no padded copy of the input exists.
struct ConvGeom {
    int taps;     // 0 (GEMM), 9 (3x3)
    int cblocks;  // C_in / 64
    int W;        // OUTPUT width
    int HW;       // OUTPUT height * width
    int stride;   // 1 or 2 (the tensor map carries the matching element strides)
    // Batched GEMM (taps == 0, batch_m > 0): the M rows are batch_m-row groups; group g multiplies against ITS OWN
    // block of W rows, [g * b_batch_rows, g * b_batch_rows + N)  - e.g. S_g = Q_g K_g^T per image.  a_mod > 0: the A
    // operand is shared by all groups (A row = row % a_mod) - e.g. V_g^T = W_v X_g^T.  batch_m % 128 == 0, N % 256 == 0.
    int batch_m = 0;
    int a_mod = 0;
    int b_batch_rows = 0;
    int pad = 1;  // tap origin of a convolution (taps == 9): 1 or 0
};

constexpr int kGemmBlockM = 128;
constexpr int kGemmBlockK = 64;  // 64 bf16 = one 128-byte swizzle row (128 e4m3: gemm_block_k)
constexpr int kGemmThreads = 384;
constexpr int kGemmBoxRows = 128;  // rows of the TMA box of both operand tensor maps
constexpr int kGemmOutRows = 64;   // rows of an output sub-tile (one consumer warp group) and of the output tensor map's box
constexpr int kGemmOutBytes = kGemmOutRows * 128;  // one staging buffer: 64 rows of 128 bytes (64 bf16 / 32 fp32 columns)

// K elements of one slab (one 128-byte swizzle row) of operand type Op.
template <typename Op>
__host__ __device__ constexpr int gemm_block_k() { return 128 / static_cast<int>(sizeof(Op)); }

template <int BN>
struct GemmCfg {
    static constexpr int kABytes = kGemmBlockM * kGemmBlockK * 2;
    static constexpr int kBBytes = BN * kGemmBlockK * 2;
    static constexpr int kStageBytes = kABytes + kBBytes;
    static constexpr int kStages = (BN == 256) ? 4 : 6;  // 192 KB of operand slabs
    static constexpr int kOutBytes = 2 * 2 * kGemmOutBytes;  // two staging buffers per consumer warp group: 32 KB
    static constexpr int kSmemBytes = kStages * kStageBytes + kOutBytes + 1024 /*align slack*/ + 256 /*barriers*/;
    static_assert(kSmemBytes <= 227 * 1024, "more shared memory than an sm_90 block may have");
};

// ------------------------------------------------------------------------------------------------
// wgmma (sm_90a)

// Shared-memory matrix descriptor of a K-major operand in 128-byte swizzle (layout type 1 at bits [62,64)): rows of
// 64 bf16 = 128 B, 8-row atoms of 1024 B => SBO = 1024 B; LBO is unused for this layout.  Stage buffers are 1024-aligned.
LFM_DEVICE uint64_t make_wgmma_desc_sw128(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
    d |= static_cast<uint64_t>(1) << 16;
    d |= static_cast<uint64_t>(1024 >> 4) << 32;
    d |= 1ull << 62;
    return d;
}
LFM_DEVICE void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
LFM_DEVICE void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
LFM_DEVICE void wgmma_wait() {
    asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accesses of the accumulator registers across the asynchronous wgmma window
LFM_DEVICE void fence_operand(float& r) { asm volatile("" : "+f"(r)::"memory"); }

// The accumulator operands of one wgmma: N / 2 fp32 registers per thread of the warp group (N = 128 or 256).
#define LFM_WGMMA_ACC64 \
    "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, " \
    "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, " \
    "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, " \
    "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
#define LFM_WGMMA_ACC128 \
    "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, " \
    "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, " \
    "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, " \
    "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, " \
    "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, " \
    "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, " \
    "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, " \
    "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"
#define LFM_WGMMA_ACC64_OPS(d) \
    "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), \
    "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), \
    "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), \
    "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), \
    "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), \
    "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), \
    "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), \
    "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
#define LFM_WGMMA_ACC128_OPS(d) \
    "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), \
    "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), \
    "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), \
    "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), \
    "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), \
    "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), \
    "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), \
    "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), \
    "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), \
    "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), \
    "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), \
    "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), \
    "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), \
    "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), \
    "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), \
    "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])

// D[64 x 256] (fp32, registers) += A[64 x 16] (smem) * B[256 x 16]^T (smem), both K-major bf16
LFM_DEVICE void wgmma_m64n256k16(float* d, uint64_t desc_a, uint64_t desc_b) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {" LFM_WGMMA_ACC128 "}, %128, %129, p, 1, 1, 0, 0;\n\t}"
        : LFM_WGMMA_ACC128_OPS(d)
        : "l"(desc_a), "l"(desc_b), "r"(1));
}

// D[64 x 128] (fp32, registers) += A[64 x 16] (smem) * B[128 x 16]^T (smem), both K-major bf16
LFM_DEVICE void wgmma_m64n128k16(float* d, uint64_t desc_a, uint64_t desc_b) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {" LFM_WGMMA_ACC64 "}, %64, %65, p, 1, 1, 0, 0;\n\t}"
        : LFM_WGMMA_ACC64_OPS(d)
        : "l"(desc_a), "l"(desc_b), "r"(1));
}

// D[64 x 256] += A[64 x 32] * B[256 x 32]^T, both K-major e4m3 (FP8 wgmma takes no transpose operands: K-major only)
LFM_DEVICE void wgmma_m64n256k32_e4m3(float* d, uint64_t desc_a, uint64_t desc_b) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k32.f32.e4m3.e4m3 {" LFM_WGMMA_ACC128 "}, %128, %129, p, 1, 1;\n\t}"
        : LFM_WGMMA_ACC128_OPS(d)
        : "l"(desc_a), "l"(desc_b), "r"(1));
}

// D[64 x 128] += A[64 x 32] * B[128 x 32]^T, both K-major e4m3
LFM_DEVICE void wgmma_m64n128k32_e4m3(float* d, uint64_t desc_a, uint64_t desc_b) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k32.f32.e4m3.e4m3 {" LFM_WGMMA_ACC64 "}, %64, %65, p, 1, 1;\n\t}"
        : LFM_WGMMA_ACC64_OPS(d)
        : "l"(desc_a), "l"(desc_b), "r"(1));
}

// One 32-byte K step of a 64 x BN tile: k16 for bf16 operands, k32 for e4m3.
template <int BN, typename Op>
LFM_DEVICE void wgmma_tile(float* d, uint64_t desc_a, uint64_t desc_b) {
    if constexpr (std::is_same_v<Op, __nv_fp8_e4m3>) {
        if constexpr (BN == 256)
            wgmma_m64n256k32_e4m3(d, desc_a, desc_b);
        else
            wgmma_m64n128k32_e4m3(d, desc_a, desc_b);
    } else {
        if constexpr (BN == 256)
            wgmma_m64n256k16(d, desc_a, desc_b);
        else
            wgmma_m64n128k16(d, desc_a, desc_b);
    }
}

LFM_DEVICE void tma_load_4d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int32_t c0, int32_t c1, int32_t c2, int32_t c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}

// Butterfly sum over the lanes that differ in the bits >= first_off of the lane index (every lane keeps the result).
LFM_DEVICE float warp_sum_mask(float v, int first_off) {
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1)
        if (o >= first_off) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
LFM_DEVICE void gn_add(unsigned long long* bins_b, int g, float s, float q) {
    atomicAdd(bins_b + 2 * g, static_cast<unsigned long long>(__double2ll_rn(static_cast<double>(s) * kGnFixScale)));
    atomicAdd(bins_b + 2 * g + 1, static_cast<unsigned long long>(__double2ll_rn(static_cast<double>(q) * kGnFixScaleSq)));
}

// 4 x 4 transpose of 32-bit items within each quad of lanes (q = lane % 4): a[i] of lane q becomes a[q] of lane i.
LFM_DEVICE void quad_transpose(uint32_t (&a)[4]) {
    const int lane = threadIdx.x & 31, q = lane & 3;
    uint32_t b[4];
#pragma unroll
    for (int s = 0; s < 4; ++s) b[s] = (s == q) ? a[s] : 0u;
#pragma unroll
    for (int k = 1; k < 4; ++k) {
        const int send = (q + k) & 3, from = (q - k) & 3;  // lane q sends its item for lane q + k, receives from lane q - k
        const uint32_t v = send == 0 ? a[0] : send == 1 ? a[1] : send == 2 ? a[2] : a[3];
        const uint32_t r = __shfl_sync(0xffffffffu, v, (lane & ~3) | from);
#pragma unroll
        for (int s = 0; s < 4; ++s)
            if (s == from) b[s] = r;
    }
#pragma unroll
    for (int s = 0; s < 4; ++s) a[s] = b[s];
}

// Epilogue of 32 whole columns c32 .. c32 + 31 (in range, 16-byte aligned rows) from acc[0, 16) of the accumulator layout:
// the same arithmetic per element as the per-8-column path, then a quad transpose so that lane q holds columns
// c32 + 8 q .. + 7 of its two rows and stores them with 16-byte accesses.
template <int EPI>
LFM_DEVICE void epilogue_store_32(const float* acc, const GemmEpi& ep, int c32, bool ok0, bool ok1, int row0, int row1, int orow0,
                                  int orow1, const float* gate0, const float* gate1) {
    const int q = threadIdx.x & 3;
    uint32_t r0a[4], r0b[4], r1a[4], r1b[4];  // bf16: packed pairs in r0a / r1a; fp32: .x in *a, .y in *b
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int col = c32 + 8 * k + 2 * q;
        float v0 = acc[4 * k], v1 = acc[4 * k + 1], v2 = acc[4 * k + 2], v3 = acc[4 * k + 3];
        if (ep.bias != nullptr) {
            const float b0 = __ldg(ep.bias + col), b1 = __ldg(ep.bias + col + 1);
            v0 += b0, v1 += b1, v2 += b0, v3 += b1;
        }
        if (EPI == EPI_BIAS_GELU_BF16) {
            v0 = gelu_tanh(v0), v1 = gelu_tanh(v1), v2 = gelu_tanh(v2), v3 = gelu_tanh(v3);
        }
        if (EPI == EPI_BIAS_BF16 || EPI == EPI_BIAS_GELU_BF16) {
            r0a[k] = pack_bf16x2(v0, v1);
            r1a[k] = pack_bf16x2(v2, v3);
        } else {
            r0a[k] = __float_as_uint(v0), r0b[k] = __float_as_uint(v1);
            r1a[k] = __float_as_uint(v2), r1b[k] = __float_as_uint(v3);
        }
    }
    const int col = c32 + 8 * q;  // this lane's 8 columns after the transpose; item p = columns col + 2 p, + 1
    if (EPI == EPI_BIAS_BF16 || EPI == EPI_BIAS_GELU_BF16) {
        quad_transpose(r0a);
        quad_transpose(r1a);
        __nv_bfloat16* o = static_cast<__nv_bfloat16*>(ep.out);
        if (ok0) *reinterpret_cast<uint4*>(o + static_cast<size_t>(orow0) * ep.ldo + col) = make_uint4(r0a[0], r0a[1], r0a[2], r0a[3]);
        if (ok1) *reinterpret_cast<uint4*>(o + static_cast<size_t>(orow1) * ep.ldo + col) = make_uint4(r1a[0], r1a[1], r1a[2], r1a[3]);
        return;
    }
    quad_transpose(r0a);
    quad_transpose(r0b);
    quad_transpose(r1a);
    quad_transpose(r1b);
    float* o = static_cast<float*>(ep.out);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const bool ok = h == 0 ? ok0 : ok1;
        if (!ok) continue;
        const uint32_t* ra = h == 0 ? r0a : r1a;
        const uint32_t* rb = h == 0 ? r0b : r1b;
        float v[8];
#pragma unroll
        for (int p = 0; p < 4; ++p) v[2 * p] = __uint_as_float(ra[p]), v[2 * p + 1] = __uint_as_float(rb[p]);
        if (EPI == EPI_BIAS_F32) {
            float4* d = reinterpret_cast<float4*>(o + static_cast<size_t>(h == 0 ? orow0 : orow1) * ep.ldo + col);
            d[0] = make_float4(v[0], v[1], v[2], v[3]);
            d[1] = make_float4(v[4], v[5], v[6], v[7]);
        } else {  // EPI_GATE_RESID_F32
            float4* d = reinterpret_cast<float4*>(o + static_cast<size_t>(h == 0 ? row0 : row1) * ep.ldo + col);
            const float* g = h == 0 ? gate0 : gate1;
            float4 x0 = d[0], x1 = d[1];
            float* x = reinterpret_cast<float*>(&x0);
            float* y = reinterpret_cast<float*>(&x1);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (g != nullptr) {
                    x[j] = fmaf(__ldg(g + col + j), v[j], x[j]);
                    y[j] = fmaf(__ldg(g + col + 4 + j), v[4 + j], y[j]);
                } else {
                    x[j] += v[j];
                    y[j] += v[4 + j];
                }
            }
            d[0] = x0;
            d[1] = x1;
        }
    }
}

// Epilogue of one consumer warp group's 64 rows (grow .. grow + 63, all < M) through shared memory: the BN columns go out in
// sub-tiles of 128 bytes per row (64 bf16 / 32 fp32 columns), each staged in one of the group's two buffers `sc` in the
// output map's 128-byte swizzle (16-byte chunk c of row r at chunk c ^ (r % 8)) and written by one TMA store, which drains
// while the group fills the other buffer.  The residual stream's sub-tile is TMA-loaded into its buffer one sub-tile ahead
// (the first one before the main loop), updated in place and stored back.  Per element the arithmetic is the register path's.
// `obuf` (the buffer of the next sub-tile) and `xphase` (parity bit per buffer of the load barriers `xb`) carry over tiles.
template <int BN, int EPI>
LFM_DEVICE void epilogue_tma(const float* acc, const GemmEpi& ep, const CUtensorMap* tmap_c, uint8_t* sc, uint64_t* xb, int& obuf,
                             uint32_t& xphase, int grow, int nbase, int N, int bar_id) {
    constexpr bool kBf16 = EPI == EPI_BIAS_BF16 || EPI == EPI_BIAS_GELU_BF16;
    constexpr int kCols = kBf16 ? 64 : 32;
    const int lane = threadIdx.x & 31, q = lane & 3, warp_in = (threadIdx.x >> 5) & 3;
    const bool leader = (threadIdx.x & 127) == 0;
    const int r0 = warp_in * 16 + (lane >> 2);  // this lane's rows r0, r0 + 8 of the sub-tile; both are (lane / 4) mod 8
    const float* gate0 = nullptr;
    const float* gate1 = nullptr;
    if (EPI == EPI_GATE_RESID_F32 && ep.gate != nullptr) {
        gate0 = ep.gate + static_cast<size_t>((grow + r0) / ep.rows_per_sample) * ep.gate_stride;
        gate1 = ep.gate + static_cast<size_t>((grow + r0 + 8) / ep.rows_per_sample) * ep.gate_stride;
    }
#pragma unroll
    for (int s = 0; s < BN / kCols; ++s) {
        const int c0 = nbase + s * kCols;  // warp-uniform
        if (c0 >= N) break;
        uint8_t* buf = sc + obuf * kGemmOutBytes;
        if (EPI == EPI_GATE_RESID_F32) {
            if (leader) {
                tma_store_wait_read<0>();  // the other buffer's store (the previous sub-tile) has read it
                if (s + 1 < BN / kCols && c0 + kCols < N) {
                    mbar_arrive_expect_tx(&xb[obuf ^ 1], kGemmOutBytes);
                    tma_load_2d(sc + (obuf ^ 1) * kGemmOutBytes, tmap_c, &xb[obuf ^ 1], c0 + kCols, grow);
                }
            }
            mbar_wait(&xb[obuf], (xphase >> obuf) & 1u);
            xphase ^= 1u << obuf;
        } else {
            if (leader) tma_store_wait_read<1>();  // the store issued from this buffer two sub-tiles ago has read it
            named_bar_sync(bar_id, 128);
        }
        const uint32_t base = smem_u32(buf);
        if constexpr (kBf16) {
#pragma unroll
            for (int p = 0; p < 4; ++p) {
                uint32_t rr[4];
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int i = s * 8 + 2 * p + h;
                    const int col = nbase + 8 * i + 2 * q;
                    float v0 = acc[4 * i], v1 = acc[4 * i + 1], v2 = acc[4 * i + 2], v3 = acc[4 * i + 3];
                    if (ep.bias != nullptr && col < N) {
                        const float b0 = __ldg(ep.bias + col), b1 = __ldg(ep.bias + col + 1);
                        v0 += b0, v1 += b1, v2 += b0, v3 += b1;
                    }
                    if (EPI == EPI_BIAS_GELU_BF16) {
                        v0 = gelu_tanh(v0), v1 = gelu_tanh(v1), v2 = gelu_tanh(v2), v3 = gelu_tanh(v3);
                    }
                    rr[2 * h] = pack_bf16x2(v0, v1);
                    rr[2 * h + 1] = pack_bf16x2(v2, v3);
                }
                // matrix m = lane / 8: rows + 8 (m & 1), chunk 2 p + m / 2
                const int m = lane >> 3, row = warp_in * 16 + (m & 1) * 8 + (lane & 7), chunk = 2 * p + (m >> 1);
                stmatrix_x4(base + row * 128 + ((chunk ^ (lane & 7)) << 4), rr[0], rr[1], rr[2], rr[3]);
            }
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int i = s * 4 + j;
                const int col = nbase + 8 * i + 2 * q;
                if (col >= N) continue;  // past the tail: the TMA store clips these columns
                float v0 = acc[4 * i], v1 = acc[4 * i + 1], v2 = acc[4 * i + 2], v3 = acc[4 * i + 3];
                if (ep.bias != nullptr) {
                    const float b0 = __ldg(ep.bias + col), b1 = __ldg(ep.bias + col + 1);
                    v0 += b0, v1 += b1, v2 += b0, v3 += b1;
                }
                const int off = (((2 * j + (q >> 1)) ^ ((lane >> 2) & 7)) << 4) + 8 * (q & 1);
                float2* p0 = reinterpret_cast<float2*>(buf + r0 * 128 + off);
                float2* p1 = reinterpret_cast<float2*>(buf + (r0 + 8) * 128 + off);
                if (EPI == EPI_BIAS_F32) {
                    *p0 = make_float2(v0, v1);
                    *p1 = make_float2(v2, v3);
                } else {
                    float2 x = *p0, y = *p1;
                    if (gate0 != nullptr) {
                        x.x = fmaf(__ldg(gate0 + col), v0, x.x);
                        x.y = fmaf(__ldg(gate0 + col + 1), v1, x.y);
                        y.x = fmaf(__ldg(gate1 + col), v2, y.x);
                        y.y = fmaf(__ldg(gate1 + col + 1), v3, y.y);
                    } else {
                        x.x += v0, x.y += v1, y.x += v2, y.y += v3;
                    }
                    *p0 = x;
                    *p1 = y;
                }
            }
        }
        fence_proxy_async();  // the generic-proxy writes above, before the TMA store reads them
        named_bar_sync(bar_id, 128);
        if (leader) {
            tma_store_2d(tmap_c, buf, c0, grow);
            tma_store_commit();
        }
        obuf ^= 1;
    }
}

// Work items: (tile, k-slice).  ksplit > 1 (split-K, for GEMMs with far fewer tiles than SMs): every slice stores its fp32
// partial tile, without bias, into its own slab of ep.out (row offset slice * split_row_pitch); a separate kernel adds the
// slabs in a fixed order.
template <int BN, int EPI, typename Op = __nv_bfloat16>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_bf16_wgmma(const __grid_constant__ CUtensorMap tmap_a,  // A [M, K] (or the 4-D NHWC activation of a convolution), box 128 rows
                const __grid_constant__ CUtensorMap tmap_b,  // W [N, K], box {64, 128}
                const __grid_constant__ CUtensorMap tmap_c,  // out, when ep.out_map != nullptr (make_tmap_out)
                int M, int N, int K, GemmEpi ep, ConvGeom cg, int ksplit, int split_row_pitch) {
    using Cfg = GemmCfg<BN>;
    constexpr int kStages = Cfg::kStages;
    constexpr bool kFp8 = std::is_same_v<Op, __nv_fp8_e4m3>;
    constexpr int kBlockK = gemm_block_k<Op>();
    static_assert(!kFp8 || EPI == EPI_BIAS_BF16 || EPI == EPI_BIAS_GELU_BF16, "FP8 operands: the bf16-output epilogues only");
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* smem_a = smem;
    uint8_t* smem_b = smem + kStages * Cfg::kABytes;
    uint8_t* smem_c = smem + kStages * Cfg::kStageBytes;  // [consumer group][2] staging buffers of the TMA-store epilogue
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem_c + Cfg::kOutBytes);
    uint64_t* full_bar = bars;                 // [kStages] TMA -> consumers
    uint64_t* empty_bar = bars + kStages;      // [kStages] consumers (8 warps) -> TMA
    uint64_t* x_bar = bars + 2 * kStages;      // [consumer group][2] residual-stream sub-tile loaded into a staging buffer

    const int wg = threadIdx.x >> 7;
    const int lane = threadIdx.x & 31;

    const int n_blocks = (N + BN - 1) / BN;
    const int m_blocks = (M + kGemmBlockM - 1) / kGemmBlockM;
    const int num_items = m_blocks * n_blocks * ksplit;
    const int num_kb = K / kBlockK;
    const int kb_per = (num_kb + ksplit - 1) / ksplit;
    auto decode = [&](int item, int& m_blk, int& n_blk, int& ks) {
        const int tile = item / ksplit;
        ks = item - tile * ksplit;
        m_blk = tile / n_blocks;
        n_blk = tile - m_blk * n_blocks;
        if (ep.reverse_m) m_blk = m_blocks - 1 - m_blk;
    };

    if (threadIdx.x == 0) {
        prefetch_tmap(&tmap_a);
        prefetch_tmap(&tmap_b);
        if (ep.out_map != nullptr) prefetch_tmap(&tmap_c);
        for (int s = 0; s < kStages; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], 8);
        }
        for (int s = 0; s < 4; ++s) mbar_init(&x_bar[s], 1);
        fence_barrier_init();
        fence_proxy_async();
    }
    __syncthreads();
    pdl_wait();  // everything above overlapped the tail of the previous kernel; its outputs are complete from here on
    pdl_trigger();

    if (wg == 0) {
        // ===================== TMA producer =====================
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
        if (threadIdx.x == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
                int m_blk, n_blk, ks;
                decode(item, m_blk, n_blk, ks);
                const int row_v = m_blk * kGemmBlockM;
                const int row_a = cg.a_mod > 0 ? row_v % cg.a_mod : row_v;
                const int row_b = (cg.batch_m > 0 ? (row_v / cg.batch_m) * cg.b_batch_rows : 0) + n_blk * BN;
                int img0 = 0, h0 = 0, w0 = 0;
                if (cg.taps != 0) {
                    img0 = row_a / cg.HW;
                    h0 = (row_a % cg.HW) / cg.W;
                    w0 = row_a % cg.W;  // non-zero only when an image row is wider than the 128-pixel tile (W = 256, 512)
                }
                const int kb0 = ks * kb_per, kb1 = min(num_kb, kb0 + kb_per);
                int tap = 0, cb = 0;
                if (cg.taps != 0) {
                    tap = kb0 / cg.cblocks;
                    cb = kb0 % cg.cblocks;
                }
                for (int kb = kb0; kb < kb1; ++kb) {
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    mbar_arrive_expect_tx(&full_bar[stage], Cfg::kStageBytes);
                    uint8_t* sa = smem_a + stage * Cfg::kABytes;
                    if (cg.taps == 0) {
                        tma_load_2d(sa, &tmap_a, &full_bar[stage], kb * kBlockK, row_a);
                    } else {
                        const int r = tap / 3, sx = tap - 3 * r;
                        tma_load_4d(sa, &tmap_a, &full_bar[stage], cb * 64, cg.stride * w0 + sx - cg.pad, cg.stride * h0 + r - cg.pad, img0);
                        if (++cb == cg.cblocks) {
                            cb = 0;
                            ++tap;
                        }
                    }
#pragma unroll
                    for (int h = 0; h < BN / kGemmBoxRows; ++h)
                        tma_load_2d(smem_b + stage * Cfg::kBBytes + h * kGemmBoxRows * 128, &tmap_b, &full_bar[stage], kb * kBlockK,
                                    row_b + h * kGemmBoxRows);
                    if (++stage == kStages) {
                        stage = 0;
                        phase ^= 1;
                    }
                }
            }
        }
    } else {
        // ===================== consumers: rows 64 (wg - 1) .. + 64 of the tile =====================
        asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory");
        const int cw = wg - 1;
        const int warp_in = (threadIdx.x >> 5) & 3;
        float acc[BN / 2];
        int stage = 0;
        uint32_t phase = 0;
        uint8_t* sc = smem_c + cw * 2 * kGemmOutBytes;
        uint64_t* xb = x_bar + 2 * cw;
        int obuf = 0;
        uint32_t xphase = 0;
        const bool leader = (threadIdx.x & 127) == 0;
        for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
            int m_blk, n_blk, ks;
            decode(item, m_blk, n_blk, ks);
            const int kb0 = ks * kb_per, kb1 = min(num_kb, kb0 + kb_per);
            const int grow = m_blk * kGemmBlockM + cw * 64;  // first row of this warp group
            const bool tma_epi = ep.out_map != nullptr && grow + kGemmOutRows <= M;  // warp-group-uniform
            if (EPI == EPI_GATE_RESID_F32 && tma_epi && leader) {  // the first residual sub-tile loads under the main loop
                tma_store_wait_read<0>();
                mbar_arrive_expect_tx(&xb[obuf], kGemmOutBytes);
                tma_load_2d(sc + obuf * kGemmOutBytes, &tmap_c, &xb[obuf], n_blk * BN, grow);
            }
#pragma unroll
            for (int j = 0; j < BN / 2; ++j) acc[j] = 0.f;
            int prev_stage = 0;
            for (int kb = kb0; kb < kb1; ++kb) {
                mbar_wait(&full_bar[stage], phase);
#pragma unroll
                for (int j = 0; j < BN / 2; ++j) fence_operand(acc[j]);
                wgmma_fence();
                const uint64_t da = make_wgmma_desc_sw128(smem_u32(smem_a + stage * Cfg::kABytes + cw * 64 * 128));
                const uint64_t db = make_wgmma_desc_sw128(smem_u32(smem_b + stage * Cfg::kBBytes));
#pragma unroll
                for (int k = 0; k < 4; ++k) wgmma_tile<BN, Op>(acc, da + 2 * k, db + 2 * k);  // +32 B per K step (16 bf16 / 32 e4m3)
                wgmma_commit();
                wgmma_wait<1>();  // the previous slab's MMAs are complete: its slot can be refilled
#pragma unroll
                for (int j = 0; j < BN / 2; ++j) fence_operand(acc[j]);
                if (kb > kb0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);
                prev_stage = stage;
                if (++stage == kStages) {
                    stage = 0;
                    phase ^= 1;
                }
            }
            wgmma_wait<0>();
#pragma unroll
            for (int j = 0; j < BN / 2; ++j) fence_operand(acc[j]);
            if (kb1 > kb0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);
            if constexpr (kFp8) {  // dequantise: acc[4 i + {0, 1}] is row r0, acc[4 i + {2, 3}] row r0 + 8 (layout below)
                const int r0 = m_blk * kGemmBlockM + cw * 64 + warp_in * 16 + (lane >> 2);
                const float sa0 = __ldg(ep.a_scale + min(r0, M - 1)), sa1 = __ldg(ep.a_scale + min(r0 + 8, M - 1));
#pragma unroll
                for (int i = 0; i < BN / 8; ++i) {
                    const int col = n_blk * BN + 8 * i + 2 * (lane & 3);
                    if (col < N) {  // N is even
                        const float sw0 = __ldg(ep.w_scale + col), sw1 = __ldg(ep.w_scale + col + 1);
                        acc[4 * i] = acc[4 * i] * sa0 * sw0;
                        acc[4 * i + 1] = acc[4 * i + 1] * sa0 * sw1;
                        acc[4 * i + 2] = acc[4 * i + 2] * sa1 * sw0;
                        acc[4 * i + 3] = acc[4 * i + 3] * sa1 * sw1;
                    }
                }
            }
            if (tma_epi) {
                epilogue_tma<BN, EPI>(acc, ep, &tmap_c, sc, xb, obuf, xphase, grow, n_blk * BN, N, 1 + cw);
                continue;
            }

            // ---- epilogue from registers.  wgmma accumulator layout: acc[4 i + {0, 1}] = row r0, columns 8 i + 2 (lane % 4) + {0, 1};
            // acc[4 i + {2, 3}] = row r0 + 8, same columns; r0 = 16 warp + lane / 4 within the warp group's 64 rows.
            const int wrow = m_blk * kGemmBlockM + cw * 64 + warp_in * 16;  // first row of this warp
            const int row0 = wrow + (lane >> 2), row1 = row0 + 8;
            const bool ok0 = row0 < M, ok1 = row1 < M;
            const int orow0 = row0 + ks * split_row_pitch, orow1 = row1 + ks * split_row_pitch;
            const int nbase = n_blk * BN;
            const float* gate0 = nullptr;
            const float* gate1 = nullptr;
            if (EPI == EPI_GATE_RESID_F32 && ep.gate != nullptr) {
                gate0 = ep.gate + static_cast<size_t>((ok0 ? row0 : M - 1) / ep.rows_per_sample) * ep.gate_stride;
                gate1 = ep.gate + static_cast<size_t>((ok1 ? row1 : M - 1) / ep.rows_per_sample) * ep.gate_stride;
            }
            const bool gn = (EPI == EPI_BIAS_F32 || EPI == EPI_BIAS_BF16) && ep.gn_bins != nullptr && wrow < M;
            unsigned long long* bins_b = nullptr;
            if (gn) {
                const int rep = static_cast<int>((blockIdx.x * 5u + (threadIdx.x >> 5)) % kGnBinReplicas);
                bins_b = ep.gn_bins + (static_cast<size_t>(wrow / ep.gn_hw) * kGnBinReplicas + rep) * 64;
            }
            float gs = 0.f, gq = 0.f;
            // Whole 32-column groups are stored 16 bytes per lane (a quad of lanes writes 64 contiguous bytes of a row, 128 for
            // fp32) after a transpose within the quad; the per-8-column path below takes the N tail, the GroupNorm statistics and
            // rows whose pitch or base is not 16-byte aligned.
            const bool vec = !gn && ep.ldo % 8 == 0 && (reinterpret_cast<uintptr_t>(ep.out) & 15) == 0;
#pragma unroll
            for (int i4 = 0; i4 < BN / 8; i4 += 4) {
                const int c32 = nbase + 8 * i4;  // warp-uniform
                if (c32 >= N) break;
                if (vec && c32 + 32 <= N) {
                    epilogue_store_32<EPI>(acc + 4 * i4, ep, c32, ok0, ok1, row0, row1, orow0, orow1, gate0, gate1);
                    continue;
                }
#pragma unroll
                for (int i = i4; i < i4 + 4; ++i) {
                    const int c8 = nbase + 8 * i;  // warp-uniform
                    if (c8 >= N) break;
                    const int col = c8 + 2 * (lane & 3);
                    const bool cok = col < N;  // N is even; a tail narrower than 8 columns (N = 4) ends inside the block
                    const bool w0 = ok0 && cok, w1 = ok1 && cok;
                    float v0 = acc[4 * i], v1 = acc[4 * i + 1], v2 = acc[4 * i + 2], v3 = acc[4 * i + 3];
                    if (ep.bias != nullptr && cok) {
                        const float b0 = __ldg(ep.bias + col), b1 = __ldg(ep.bias + col + 1);
                        v0 += b0, v1 += b1, v2 += b0, v3 += b1;
                    }
                    if (EPI == EPI_BIAS_GELU_BF16) {
                        v0 = gelu_tanh(v0), v1 = gelu_tanh(v1), v2 = gelu_tanh(v2), v3 = gelu_tanh(v3);
                    }
                    if (EPI == EPI_BIAS_BF16 || EPI == EPI_BIAS_GELU_BF16) {
                        __nv_bfloat16* o = static_cast<__nv_bfloat16*>(ep.out);
                        if (w0) *reinterpret_cast<uint32_t*>(o + static_cast<size_t>(orow0) * ep.ldo + col) = pack_bf16x2(v0, v1);
                        if (w1) *reinterpret_cast<uint32_t*>(o + static_cast<size_t>(orow1) * ep.ldo + col) = pack_bf16x2(v2, v3);
                    } else if (EPI == EPI_BIAS_F32) {
                        float* o = static_cast<float*>(ep.out);
                        if (w0) *reinterpret_cast<float2*>(o + static_cast<size_t>(orow0) * ep.ldo + col) = make_float2(v0, v1);
                        if (w1) *reinterpret_cast<float2*>(o + static_cast<size_t>(orow1) * ep.ldo + col) = make_float2(v2, v3);
                    } else {  // EPI_GATE_RESID_F32
                        float* o = static_cast<float*>(ep.out);
                        if (w0) {
                            float2* p = reinterpret_cast<float2*>(o + static_cast<size_t>(row0) * ep.ldo + col);
                            float2 x = *p;
                            if (gate0 != nullptr) {
                                x.x = fmaf(__ldg(gate0 + col), v0, x.x);
                                x.y = fmaf(__ldg(gate0 + col + 1), v1, x.y);
                            } else {
                                x.x += v0, x.y += v1;
                            }
                            *p = x;
                        }
                        if (w1) {
                            float2* p = reinterpret_cast<float2*>(o + static_cast<size_t>(row1) * ep.ldo + col);
                            float2 x = *p;
                            if (gate1 != nullptr) {
                                x.x = fmaf(__ldg(gate1 + col), v2, x.x);
                                x.y = fmaf(__ldg(gate1 + col + 1), v3, x.y);
                            } else {
                                x.x += v2, x.y += v3;
                            }
                            *p = x;
                        }
                    }
                    if (EPI == EPI_BIAS_F32 || EPI == EPI_BIAS_BF16) {
                        if (gn) {  // warp-uniform
                            if (!w0) v0 = v1 = 0.f;
                            if (!w1) v2 = v3 = 0.f;
                            gs += (v0 + v1) + (v2 + v3);
                            gq += (v0 * v0 + v1 * v1) + (v2 * v2 + v3 * v3);
                            if (ep.gn_cpg == 4) {
                                // two groups in these 8 columns: lanes with lane % 4 in {0, 1} hold group 2 i, {2, 3} group 2 i + 1
                                const float s4 = warp_sum_mask(gs, 4), q4 = warp_sum_mask(gq, 4);
                                const float s = s4 + __shfl_xor_sync(0xffffffffu, s4, 1), q = q4 + __shfl_xor_sync(0xffffffffu, q4, 1);
                                if ((lane & ~2) == 0) gn_add(bins_b, col / 4, s, q);
                                gs = gq = 0.f;
                            } else if (((8 * (i + 1)) % ep.gn_cpg) == 0) {  // last 8 columns of a group
                                const float s = warp_sum_mask(gs, 1), q = warp_sum_mask(gq, 1);
                                if (lane == 0) gn_add(bins_b, c8 / ep.gn_cpg, s, q);
                                gs = gq = 0.f;
                            }
                        }
                    }
                }
            }
        }
        if (leader) tma_store_wait<0>();  // the stores are complete (not only read) before the grid can count as finished
    }
}

}  // namespace lfm
