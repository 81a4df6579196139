// lfm_b200 - flash-style attention on warp-level mma.sync for every DiT configuration and the long-grid UNet attention layers
// whose sequence does not fit in registers (T = 16 / 64: attention_mma_kernel, unet.cuh):
//   * 256 tokens with head_dim 64 (every released preset: /2 nets on 32 x 32 latents) and 1024-token grids (64 x 64 latents with
//     patch 2: 512-pixel images on a DiT-*/2),
//   * head_dim 72 (the DiT-XL entries of models/DiT.py:355-365) - stored padded to CH = 80 channels per head with zero weight rows,
//     so q.k and P.V are unchanged and the padded output columns are zero.
// softmax(q k^T * head_dim^-1/2) v of timm's Attention (models/DiT.py:120; SURVEY D6), keys streamed in chunks of 64 through a
// double-buffered shared-memory ring (cp.async) with the running-maximum rescaling of FlashAttention-2: one block = 64 query rows of
// one (sample, head), 4 warps x 16 rows; S = Q K_j^T (m16n8k16 bf16, fp32 accumulate) never leaves registers, the row maximum and
// the exponentials are fp32, P is rounded to bf16 as the A operand of P V_j.  Same fragment / ldmatrix index patterns as
// attention_mma_kernel.  Two qkv row layouts (row = 3 C features of one token):
//   head-major  feature = head * 3 CH + {q,k,v} * CH + c     (head_stride = 3 CH, part_stride = CH; re-ordered once at lfm_set_param)
//   timm        feature = {q,k,v} * C + head * CH + c        (head_stride = CH,   part_stride = C: the checkpoint's own order)
#pragma once
#include "common.cuh"
// (ldmatrix / mma.sync / cp.async helpers: unet.cuh, included before this file by lfm_api.cu)

namespace lfm {

LFM_DEVICE void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
LFM_DEVICE void cp_async_wait_group() {
    asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

template <int CH>
__global__ void __launch_bounds__(128)
attention_flash_mma_kernel(const __nv_bfloat16* __restrict__ qkv, __nv_bfloat16* __restrict__ out, int T, int C /* heads * CH */,
                           int heads, float scale_log2e /* true head_dim^-1/2 * log2(e) */, int head_stride, int part_stride) {
    pdl_wait();
    pdl_trigger();
    static_assert(CH % 16 == 0, "head channels (padded) must be a multiple of 16");
    constexpr int LD = CH + 8;   // row pitch in elements: +16 bytes keeps ldmatrix bank-conflict free
    constexpr int CPR = CH / 8;  // 16-byte chunks per row
    constexpr int KT = 64;       // keys per chunk = query rows per block
    extern __shared__ __align__(16) uint8_t fl_smem[];
    __nv_bfloat16* sQ = reinterpret_cast<__nv_bfloat16*>(fl_smem);  // [64][LD]
    __nv_bfloat16* sK = sQ + KT * LD;                               // [2][64][LD]
    __nv_bfloat16* sV = sK + 2 * KT * LD;                           // [2][64][LD]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int q0 = blockIdx.x * KT;
    const int b = blockIdx.y / heads, h = blockIdx.y % heads;
    const size_t ld = static_cast<size_t>(3) * C;
    const __nv_bfloat16* base = qkv + static_cast<size_t>(b) * T * ld + static_cast<size_t>(h) * head_stride;
    auto load_tile = [&](__nv_bfloat16* dst, int which, int row0) {  // 64 rows x CH channels of q / k / v starting at token row0
        for (int i = threadIdx.x; i < KT * CPR; i += 128) {
            const int t = i / CPR, c8 = i % CPR;
            cp_async_16(dst + t * LD + c8 * 8, base + static_cast<size_t>(row0 + t) * ld + which * part_stride + c8 * 8);
        }
    };
    const int nchunks = T / KT;
    load_tile(sQ, 0, q0);
    load_tile(sK, 1, 0);
    load_tile(sV, 2, 0);
    cp_async_commit();

    uint32_t qf[CH / 16][4];
    float acc_o[CH / 8][4];
#pragma unroll
    for (int n = 0; n < CH / 8; ++n) acc_o[n][0] = acc_o[n][1] = acc_o[n][2] = acc_o[n][3] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;  // rows g = lane / 4 and g + 8 of this warp's 16 query rows
    const int r0 = warp * 16;

    for (int j = 0; j < nchunks; ++j) {
        const int buf = j & 1;
        if (j + 1 < nchunks) {  // prefetch the next key chunk into the other buffer (its readers finished at the end of iteration j - 1)
            load_tile(sK + (buf ^ 1) * KT * LD, 1, (j + 1) * KT);
            load_tile(sV + (buf ^ 1) * KT * LD, 2, (j + 1) * KT);
            cp_async_commit();
            cp_async_wait_group<1>();
        } else {
            cp_async_wait_group<0>();
        }
        __syncthreads();
        if (j == 0) {
#pragma unroll
            for (int kk = 0; kk < CH / 16; ++kk) ldmatrix_x4(qf[kk], sQ + (r0 + (lane & 15)) * LD + kk * 16 + (lane >> 4) * 8);
        }
        const __nv_bfloat16* sKb = sK + buf * KT * LD;
        const __nv_bfloat16* sVb = sV + buf * KT * LD;
        float acc_s[KT / 8][4];
#pragma unroll
        for (int n = 0; n < KT / 8; ++n) acc_s[n][0] = acc_s[n][1] = acc_s[n][2] = acc_s[n][3] = 0.f;
#pragma unroll
        for (int kk = 0; kk < CH / 16; ++kk) {
#pragma unroll
            for (int j2 = 0; j2 < KT / 16; ++j2) {
                uint32_t bk[4];
                ldmatrix_x4(bk, sKb + (j2 * 16 + (lane & 7) + ((lane >> 4) << 3)) * LD + kk * 16 + ((lane >> 3) & 1) * 8);
                mma_bf16_16816(acc_s[2 * j2], qf[kk], bk[0], bk[1]);
                mma_bf16_16816(acc_s[2 * j2 + 1], qf[kk], bk[2], bk[3]);
            }
        }
        // running maximum of the two rows this thread holds (a row lives in one quad of lanes)
        float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
        for (int n = 0; n < KT / 8; ++n) {
            mx0 = fmaxf(mx0, fmaxf(acc_s[n][0], acc_s[n][1]));
            mx1 = fmaxf(mx1, fmaxf(acc_s[n][2], acc_s[n][3]));
        }
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
        const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);
        const float c0 = exp2f((m0 - mn0) * scale_log2e), c1 = exp2f((m1 - mn1) * scale_log2e);  // 0 on the first chunk (m = -inf)
        m0 = mn0;
        m1 = mn1;
        l0 *= c0;
        l1 *= c1;
#pragma unroll
        for (int n = 0; n < CH / 8; ++n) {
            acc_o[n][0] *= c0;
            acc_o[n][1] *= c0;
            acc_o[n][2] *= c1;
            acc_o[n][3] *= c1;
        }
        const float ms0 = m0 * scale_log2e, ms1 = m1 * scale_log2e;
#pragma unroll
        for (int n = 0; n < KT / 8; ++n) {
            acc_s[n][0] = exp2f(fmaf(acc_s[n][0], scale_log2e, -ms0));
            acc_s[n][1] = exp2f(fmaf(acc_s[n][1], scale_log2e, -ms0));
            acc_s[n][2] = exp2f(fmaf(acc_s[n][2], scale_log2e, -ms1));
            acc_s[n][3] = exp2f(fmaf(acc_s[n][3], scale_log2e, -ms1));
            l0 += acc_s[n][0] + acc_s[n][1];  // per-thread partial row sums: the quad is reduced once, after the last chunk
            l1 += acc_s[n][2] + acc_s[n][3];
        }
#pragma unroll
        for (int kk = 0; kk < KT / 16; ++kk) {
            uint32_t pa[4];
            pa[0] = pack_bf16x2(acc_s[2 * kk][0], acc_s[2 * kk][1]);
            pa[1] = pack_bf16x2(acc_s[2 * kk][2], acc_s[2 * kk][3]);
            pa[2] = pack_bf16x2(acc_s[2 * kk + 1][0], acc_s[2 * kk + 1][1]);
            pa[3] = pack_bf16x2(acc_s[2 * kk + 1][2], acc_s[2 * kk + 1][3]);
#pragma unroll
            for (int n2 = 0; n2 < CH / 16; ++n2) {
                uint32_t bv[4];
                ldmatrix_x4_trans(bv, sVb + (kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * LD + n2 * 16 + (lane >> 4) * 8);
                mma_bf16_16816(acc_o[2 * n2], pa, bv[0], bv[1]);
                mma_bf16_16816(acc_o[2 * n2 + 1], pa, bv[2], bv[3]);
            }
        }
        __syncthreads();  // every warp is done with this buffer before the prefetch of iteration j + 1 overwrites it
    }
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
    l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    const float inv0 = 1.f / l0, inv1 = 1.f / l1;
    const int row = q0 + r0 + (lane >> 2);
    __nv_bfloat16* o0 = out + (static_cast<size_t>(b) * T + row) * C + static_cast<size_t>(h) * CH + (lane & 3) * 2;
    __nv_bfloat16* o1 = o0 + static_cast<size_t>(8) * C;
#pragma unroll
    for (int n = 0; n < CH / 8; ++n) {
        *reinterpret_cast<uint32_t*>(o0 + n * 8) = pack_bf16x2(acc_o[n][0] * inv0, acc_o[n][1] * inv0);
        *reinterpret_cast<uint32_t*>(o1 + n * 8) = pack_bf16x2(acc_o[n][2] * inv1, acc_o[n][3] * inv1);
    }
}

}  // namespace lfm
