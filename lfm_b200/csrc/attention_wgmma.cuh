// lfm_b200 - Hopper attention for 256 tokens with head_dim 64 (every released DiT preset, and the EDM 16 x 16 attention layers):
// softmax(q k^T / 8) v of timm's Attention (models/DiT.py:120) on qkv rows in the checkpoint's order ({q,k,v} * C + head * 64 + c).
//
// Persistent and warp-specialised like the GEMM (gemm.cuh).  A work item is 128 query rows of one (sample, head); warp group 0 is the
// TMA producer (one thread): Q [128 x 64], K [256 x 64] and V [256 x 64] of an item land in one stage of a 2-stage ring (80 KB each,
// 128B-swizzled), completion posted as transaction bytes on the stage's mbarrier, so the next item's tiles stream in while the current one
// is computed.  Warp groups 1 and 2 take 64 query rows each:
//   S = Q K^T        wgmma.m64n256k16, both operands K-major in shared memory, fp32 accumulators in registers (the whole key range);
//   softmax          row maximum / exponentials / row sums in fp32 registers (a row lives in one quad of lanes);
//   O = P V          wgmma.m64n64k16 with P as the register A operand (bf16, the accumulator layout of S re-packed in place) and V
//                    read MN-major from shared memory (transposed B);
// then O / rowsum is stored as bf16.  The mbarrier ring hands a stage back once all 8 consumer warps have finished their P V.
#pragma once
#include "gemm.cuh"

namespace lfm {

constexpr int kAttnT = 256;
constexpr int kAttnDh = 64;
constexpr int kAttnThreads = 384;
constexpr int kAttnStages = 2;
constexpr int kAttnQBytes = 128 * kAttnDh * 2;
constexpr int kAttnKVBytes = kAttnT * kAttnDh * 2;
constexpr int kAttnStageBytes = kAttnQBytes + 2 * kAttnKVBytes;
constexpr int kAttnSmemBytes = kAttnStages * kAttnStageBytes + 1024 /*align slack*/ + 256 /*barriers*/;

// D[64 x 64] (fp32, registers) += A[64 x 16] (bf16, registers: 4 x b32) * B[16 x 64] (smem, MN-major: imm-trans-b = 1)
LFM_DEVICE void wgmma_m64n64k16_rs_mn(float* d, const uint32_t* a, uint64_t desc_b) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
        "}, {%32, %33, %34, %35}, %36, p, 1, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(1));
}

// Shared-memory descriptor of an MN-major operand in 128-byte swizzle: 8 K-indices (rows of 64 bf16 = 128 B) per 1024-byte atom => SBO =
// 1024 B between atoms along K; the operand is exactly one 64-element atom wide along N, so LBO (the next 64 N-elements) is never used.
LFM_DEVICE uint64_t make_wgmma_desc_sw128_mn(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
    d |= static_cast<uint64_t>(8192 >> 4) << 16;
    d |= static_cast<uint64_t>(1024 >> 4) << 32;
    d |= 1ull << 62;
    return d;
}

__global__ void __launch_bounds__(kAttnThreads, 1)
attention_wgmma_t256_d64(const __grid_constant__ CUtensorMap tmap_qkv,  // qkv [rows, 3 C] bf16, box {64, 128}
                         __nv_bfloat16* __restrict__ out, int C, int heads, int n_items /* samples * heads * 2 */, float scale_log2e) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kAttnStages * kAttnStageBytes);
    uint64_t* full_bar = bars;
    uint64_t* empty_bar = bars + kAttnStages;
    const int wg = threadIdx.x >> 7;
    const int lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        prefetch_tmap(&tmap_qkv);
        for (int s = 0; s < kAttnStages; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], 8);
        }
        fence_barrier_init();
        fence_proxy_async();
    }
    __syncthreads();
    pdl_wait();
    pdl_trigger();
    if (wg == 0) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
        if (threadIdx.x == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
                const int bh = item >> 1, qb = item & 1;
                const int b = bh / heads, h = bh % heads;
                const int row0 = b * kAttnT;
                mbar_wait(&empty_bar[stage], phase ^ 1);
                mbar_arrive_expect_tx(&full_bar[stage], kAttnStageBytes);
                uint8_t* st = smem + stage * kAttnStageBytes;
                tma_load_2d(st, &tmap_qkv, &full_bar[stage], h * kAttnDh, row0 + qb * 128);
#pragma unroll
                for (int half = 0; half < 2; ++half) {
                    tma_load_2d(st + kAttnQBytes + half * 16384, &tmap_qkv, &full_bar[stage], C + h * kAttnDh, row0 + half * 128);
                    tma_load_2d(st + kAttnQBytes + kAttnKVBytes + half * 16384, &tmap_qkv, &full_bar[stage], 2 * C + h * kAttnDh,
                                row0 + half * 128);
                }
                if (++stage == kAttnStages) {
                    stage = 0;
                    phase ^= 1;
                }
            }
        }
    } else {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory");
        const int cw = wg - 1;
        const int warp_in = (threadIdx.x >> 5) & 3;
        int stage = 0;
        uint32_t phase = 0;
        for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
            const int bh = item >> 1, qb = item & 1;
            const int b = bh / heads, h = bh % heads;
            uint8_t* st = smem + stage * kAttnStageBytes;
            float s[kAttnT / 2];
#pragma unroll
            for (int j = 0; j < kAttnT / 2; ++j) s[j] = 0.f;
            mbar_wait(&full_bar[stage], phase);
#pragma unroll
            for (int j = 0; j < kAttnT / 2; ++j) fence_operand(s[j]);
            wgmma_fence();
            {
                const uint64_t dq = make_wgmma_desc_sw128(smem_u32(st + cw * 64 * 128));
                const uint64_t dk = make_wgmma_desc_sw128(smem_u32(st + kAttnQBytes));
#pragma unroll
                for (int k = 0; k < kAttnDh / 16; ++k) wgmma_m64n256k16(s, dq + 2 * k, dk + 2 * k);
            }
            wgmma_commit();
            wgmma_wait<0>();
#pragma unroll
            for (int j = 0; j < kAttnT / 2; ++j) fence_operand(s[j]);
            // softmax of rows r0 (s[4 i], s[4 i + 1]) and r0 + 8 (s[4 i + 2], s[4 i + 3])
            float m0 = -INFINITY, m1 = -INFINITY;
#pragma unroll
            for (int i = 0; i < kAttnT / 8; ++i) {
                m0 = fmaxf(m0, fmaxf(s[4 * i], s[4 * i + 1]));
                m1 = fmaxf(m1, fmaxf(s[4 * i + 2], s[4 * i + 3]));
            }
            m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 1));
            m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 2));
            m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 1));
            m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 2));
            const float ms0 = m0 * scale_log2e, ms1 = m1 * scale_log2e;
            float l0 = 0.f, l1 = 0.f;
            uint32_t p[kAttnT / 4];  // P in bf16 pairs, the A-operand layout of wgmma (one 16-key chunk = 4 registers)
#pragma unroll
            for (int i = 0; i < kAttnT / 8; ++i) {
                const float e0 = exp2f(fmaf(s[4 * i], scale_log2e, -ms0)), e1 = exp2f(fmaf(s[4 * i + 1], scale_log2e, -ms0));
                const float e2 = exp2f(fmaf(s[4 * i + 2], scale_log2e, -ms1)), e3 = exp2f(fmaf(s[4 * i + 3], scale_log2e, -ms1));
                l0 += e0 + e1;
                l1 += e2 + e3;
                p[2 * i] = pack_bf16x2(e0, e1);
                p[2 * i + 1] = pack_bf16x2(e2, e3);
            }
            l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
            l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
            l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
            l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
            float o[kAttnDh / 2];
#pragma unroll
            for (int j = 0; j < kAttnDh / 2; ++j) o[j] = 0.f;
#pragma unroll
            for (int j = 0; j < kAttnDh / 2; ++j) fence_operand(o[j]);
            wgmma_fence();
            {
                const uint32_t vbase = smem_u32(st + kAttnQBytes + kAttnKVBytes);
#pragma unroll
                for (int kc = 0; kc < kAttnT / 16; ++kc)  // 16 keys = 2048 bytes of V per step
                    wgmma_m64n64k16_rs_mn(o, p + 4 * kc, make_wgmma_desc_sw128_mn(vbase + kc * 2048));
            }
            wgmma_commit();
            wgmma_wait<0>();
#pragma unroll
            for (int j = 0; j < kAttnDh / 2; ++j) fence_operand(o[j]);
            if (lane == 0) mbar_arrive(&empty_bar[stage]);
            if (++stage == kAttnStages) {
                stage = 0;
                phase ^= 1;
            }
            const float inv0 = 1.f / l0, inv1 = 1.f / l1;
            const int row = b * kAttnT + qb * 128 + cw * 64 + warp_in * 16 + (lane >> 2);
            __nv_bfloat16* o0 = out + static_cast<size_t>(row) * C + h * kAttnDh + 2 * (lane & 3);
            __nv_bfloat16* o1 = o0 + static_cast<size_t>(8) * C;
#pragma unroll
            for (int i = 0; i < kAttnDh / 8; ++i) {
                *reinterpret_cast<uint32_t*>(o0 + 8 * i) = pack_bf16x2(o[4 * i] * inv0, o[4 * i + 1] * inv0);
                *reinterpret_cast<uint32_t*>(o1 + 8 * i) = pack_bf16x2(o[4 * i + 2] * inv1, o[4 * i + 3] * inv1);
            }
        }
    }
}

}  // namespace lfm
