// lfm_b200 - persistent, warp-specialised Hopper GEMM (TMA + mbarrier + wgmma) for every linear layer and convolution.
//
//   C[M, N] = A[M, K] * W[N, K]^T   (A: activations bf16 row-major; W: nn.Linear weight, bf16, [out, in])
//
// One 128 x BN output tile per CTA and step of a persistent tile loop (BN = 128 or 256).  Both operands are K-major,
// staged by TMA into 128B-swizzled shared memory (64-element K slabs) in a ring of kStages slots.
// Warp groups (384 threads): group 0 = TMA producer (one thread), groups 1 and 2 = consumers: each multiplies its 64 rows
// of the tile with wgmma.m64nBNk16 into registers (fp32) and applies the fused epilogue straight from those registers.
//
// Fused epilogues (reference ops they replace):
//   EPI_BIAS_BF16       out = bf16(acc + bias)                       attn.qkv       (timm Attention)
//   EPI_BIAS_GELU_BF16  out = bf16(gelu_tanh(acc + bias))            mlp.fc1 + act  (models/DiT.py:122-124)
//   EPI_GATE_RESID_F32  x  += gate[b] * (acc + bias)   (fp32 stream) attn.proj / mlp.fc2 + gated residual
//                                                                    (models/DiT.py:129-130)
//   EPI_BIAS_F32        out = addend + acc + bias (fp32)             adaLN_modulation Linears in one GEMM, convolutions
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
    // 2^28 fixed point (integer atomics => the result does not depend on the order of arrival: deterministic).  r is any of
    // kGnBinReplicas copies (chosen per warp; the consumer adds them up - integers, so still exact), so that the atomics of
    // all CTAs working on one image do not queue on the same few cache lines.  Needs gn_hw % 16 == 0.
    unsigned long long* gn_bins = nullptr;
    int gn_cpg = 0;
    int gn_hw = 1;
    // Walk the M blocks from the last to the first.  Consecutive kernels of a network alternate direction so that
    // each one starts on the rows its producer touched LAST - the part still resident in L2.
    int reverse_m = 0;
    // EPI_BIAS_F32: out = addend + acc + bias, the residual connection of a convolutional block (fp32 [M, ldo]; may alias
    // out) - so that the block's OUTPUT statistics (gn_bins) can be taken in the same epilogue.
    const float* addend = nullptr;
};
constexpr int kGnBinReplicas = 16;
constexpr double kGnFixScale = 268435456.0;  // 2^28

// Implicit-GEMM convolution geometry (taps == 0: plain GEMM, A is a 2-D [M, K] matrix).
// Output pixels are flattened (b, h, w) row-major; a tile's 128 output rows are whole image rows (W * rows == 128),
// whole images (H * W divides 128) or one 128-pixel segment of an image row (W = 256: the VAE decoder's last stage),
// so the matching input window of tap (r, s) is ONE 4-D box.
struct ConvGeom {
    int taps;     // 0 (GEMM), 9 (3x3, pad 1)
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
};

constexpr int kGemmBlockM = 128;
constexpr int kGemmBlockK = 64;  // 64 bf16 = one 128-byte swizzle row
constexpr int kGemmThreads = 384;
constexpr int kGemmBoxRows = 128;  // rows of the TMA box of both operand tensor maps

template <int BN>
struct GemmCfg {
    static constexpr int kABytes = kGemmBlockM * kGemmBlockK * 2;
    static constexpr int kBBytes = BN * kGemmBlockK * 2;
    static constexpr int kStageBytes = kABytes + kBBytes;
    static constexpr int kStages = (BN == 256) ? 4 : 6;  // 192 KB of the 227 KB a block may have
    static constexpr int kSmemBytes = kStages * kStageBytes + 1024 /*align slack*/ + 256 /*barriers*/;
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

// D[64 x 256] (fp32, registers) += A[64 x 16] (smem) * B[256 x 16]^T (smem), both K-major bf16
LFM_DEVICE void wgmma_m64n256k16(float* d, uint64_t desc_a, uint64_t desc_b) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
        "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
        "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
        "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
        "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"
        "}, %128, %129, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
          "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
          "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
          "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
          "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
          "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
          "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
          "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
          "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(desc_a), "l"(desc_b), "r"(1));
}

// D[64 x 128] (fp32, registers) += A[64 x 16] (smem) * B[128 x 16]^T (smem), both K-major bf16
LFM_DEVICE void wgmma_m64n128k16(float* d, uint64_t desc_a, uint64_t desc_b) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
        "}, %64, %65, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(desc_a), "l"(desc_b), "r"(1));
}


template <int BN>
LFM_DEVICE void wgmma_tile(float* d, uint64_t desc_a, uint64_t desc_b) {
    if constexpr (BN == 256)
        wgmma_m64n256k16(d, desc_a, desc_b);
    else
        wgmma_m64n128k16(d, desc_a, desc_b);
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
    atomicAdd(bins_b + 2 * g + 1, static_cast<unsigned long long>(__double2ll_rn(static_cast<double>(q) * kGnFixScale)));
}

// Work items: (tile, k-slice).  ksplit > 1 (split-K, for GEMMs with far fewer tiles than SMs): every slice stores its fp32
// partial tile, without bias, into its own slab of ep.out (row offset slice * split_row_pitch); a separate kernel adds the
// slabs in a fixed order.
template <int BN, int EPI>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_bf16_wgmma(const __grid_constant__ CUtensorMap tmap_a,  // A [M, K] (or the 4-D NHWC activation of a convolution), box 128 rows
                const __grid_constant__ CUtensorMap tmap_b,  // W [N, K], box {64, 128}
                int M, int N, int K, GemmEpi ep, ConvGeom cg, int ksplit, int split_row_pitch) {
    using Cfg = GemmCfg<BN>;
    constexpr int kStages = Cfg::kStages;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* smem_a = smem;
    uint8_t* smem_b = smem + kStages * Cfg::kABytes;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kStages * Cfg::kStageBytes);
    uint64_t* full_bar = bars;             // [kStages] TMA -> consumers
    uint64_t* empty_bar = bars + kStages;  // [kStages] consumers (8 warps) -> TMA

    const int wg = threadIdx.x >> 7;
    const int lane = threadIdx.x & 31;

    const int n_blocks = (N + BN - 1) / BN;
    const int m_blocks = (M + kGemmBlockM - 1) / kGemmBlockM;
    const int num_items = m_blocks * n_blocks * ksplit;
    const int num_kb = K / kGemmBlockK;
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
        for (int s = 0; s < kStages; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], 8);
        }
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
                    w0 = row_a % cg.W;  // non-zero only when an image row is wider than the 128-pixel tile (W = 256)
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
                        tma_load_2d(sa, &tmap_a, &full_bar[stage], kb * kGemmBlockK, row_a);
                    } else {
                        const int r = tap / 3, sx = tap - 3 * r;
                        tma_load_4d(sa, &tmap_a, &full_bar[stage], cb * 64, cg.stride * w0 + sx - 1, cg.stride * h0 + r - 1, img0);
                        if (++cb == cg.cblocks) {
                            cb = 0;
                            ++tap;
                        }
                    }
#pragma unroll
                    for (int h = 0; h < BN / kGemmBoxRows; ++h)
                        tma_load_2d(smem_b + stage * Cfg::kBBytes + h * kGemmBoxRows * 128, &tmap_b, &full_bar[stage], kb * kGemmBlockK,
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
        for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
            int m_blk, n_blk, ks;
            decode(item, m_blk, n_blk, ks);
            const int kb0 = ks * kb_per, kb1 = min(num_kb, kb0 + kb_per);
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
                for (int k = 0; k < kGemmBlockK / 16; ++k) wgmma_tile<BN>(acc, da + 2 * k, db + 2 * k);  // +32 B per K step of 16
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
#pragma unroll
            for (int i = 0; i < BN / 8; ++i) {
                const int c8 = nbase + 8 * i;  // warp-uniform
                if (c8 >= N) break;
                const int col = c8 + 2 * (lane & 3);
                const bool cok = col < N;  // N is even; a tail narrower than 8 columns (N = 4) ends inside the block
                const bool w0 = ok0 && cok, w1 = ok1 && cok;
                float v0 = acc[4 * i], v1 = acc[4 * i + 1], v2 = acc[4 * i + 2], v3 = acc[4 * i + 3];
                if (EPI == EPI_BIAS_F32 && ep.addend != nullptr) {
                    if (w0) {
                        const float2 a = __ldcg(reinterpret_cast<const float2*>(ep.addend + static_cast<size_t>(row0) * ep.ldo + col));
                        v0 += a.x, v1 += a.y;
                    }
                    if (w1) {
                        const float2 a = __ldcg(reinterpret_cast<const float2*>(ep.addend + static_cast<size_t>(row1) * ep.ldo + col));
                        v2 += a.x, v3 += a.y;
                    }
                }
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
}

}  // namespace lfm
