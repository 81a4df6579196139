// lfm_b200 - the non-GEMM kernels of the DiT velocity network and the ODE-solver arithmetic.
// All HBM- or latency-bound; plain CUDA cores, vectorised, coalesced.  fp32 everywhere except the bf16 tensors
// that feed the wgmma GEMMs.
#pragma once
#include "common.cuh"

namespace lfm {

// ------------------------------------------------------------------------------------------------
// The conditioning stage of every velocity network (DiT t_embedder / y_embedder, models/DiT.py:43-62,125,264; the UNets'
// time_embed / label_emb, unet.py:613-624, and map_layer0 / map_layer1 / map_label, EDM.py:812-829), per network row:
//   tf = [cos | sin](t f_k), f_k = exp(-ln(1e4) k / half)   (width 2 half, raw t, cos first; nn.py:103-121, DiT.py:43-62)
//   h1 = SiLU(W0 tf + b0)                                     (fp32)
//   c  = SiLU(W2 h1 + b2 + table[row])                        (bf16: the operand of the modulation GEMM)

// Timestep features of width dim (even); t_numel == 1 broadcasts.  One block per row.
__global__ void timestep_features_kernel(const float* __restrict__ t, int t_numel, float* __restrict__ tf, int dim) {
    pdl_wait();  // PDL: nothing of the previous kernel's output is touched above this line
    pdl_trigger();
    const int b = blockIdx.x;
    const int half = dim / 2;
    const float tv = t[t_numel == 1 ? 0 : b];
    for (int i = threadIdx.x; i < dim; i += blockDim.x) {
        const int k = i < half ? i : i - half;
        const float freq = expf(-9.210340371976184f * static_cast<float>(k) / static_cast<float>(half));
        const float a = tv * freq;
        tf[static_cast<size_t>(b) * dim + i] = (i < half) ? cosf(a) : sinf(a);
    }
}

// One MLP layer of the stage: out[b, j] = SiLU(bias[j] + W[j, :] . in[b, :] (+ table[row, j])), W [N, K] fp32, K a multiple of 128.
// One warp per output feature j: lane l accumulates the float4 m 32 + l of the row, m ascending, in one fmaf chain, then the warp
// sums.  The first kCondRegV float4 of the lane's weights stay in registers while the warp sweeps the rows; a longer row streams
// the rest from memory for every row.
//   OutT float:          SiLU -> fp32 (h1)
//   OutT __nv_bfloat16:  + the label row, SiLU -> bf16 (c).  row = idx ? clamp(idx[b], 0, max_row) : null_row; no table term
//                        when that is negative.
constexpr int kCondRegV = 9;  // K <= 1152 (every DiT width) runs from registers alone
template <typename OutT>
__global__ void __launch_bounds__(256)
condition_mlp_kernel(const float* __restrict__ W, const float* __restrict__ bias, const float* __restrict__ in, int B, int N, int K,
                     const float* __restrict__ table, const long long* __restrict__ idx, int max_row, int null_row,
                     OutT* __restrict__ out) {
    pdl_wait();  // PDL: nothing of the previous kernel's output is touched above this line
    pdl_trigger();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int j = blockIdx.x * 8 + warp;
    if (j >= N) return;
    const int nv = K / 128;  // float4 per lane
    const float4* wp = reinterpret_cast<const float4*>(W + static_cast<size_t>(j) * K) + lane;
    float4 w[kCondRegV];
#pragma unroll
    for (int m = 0; m < kCondRegV; ++m)
        if (m < nv) w[m] = __ldg(wp + m * 32);
    auto fma4 = [](float4 a, float4 x, float acc) {
        acc = fmaf(a.x, x.x, acc);
        acc = fmaf(a.y, x.y, acc);
        acc = fmaf(a.z, x.z, acc);
        return fmaf(a.w, x.w, acc);
    };
    const float bj = bias[j];
    for (int b = 0; b < B; ++b) {
        const float4* ip = reinterpret_cast<const float4*>(in + static_cast<size_t>(b) * K) + lane;
        float acc = 0.f;
#pragma unroll
        for (int m = 0; m < kCondRegV; ++m)
            if (m < nv) acc = fma4(w[m], __ldg(ip + m * 32), acc);
#pragma unroll 4  // fully unrolled, the tail's loads would take the registers of the weights above and spill
        for (int m = kCondRegV; m < nv; ++m) acc = fma4(__ldg(wp + m * 32), __ldg(ip + m * 32), acc);
        acc = warp_sum(acc);
        if (lane == 0) {
            float v = acc + bj;
            if constexpr (std::is_same_v<OutT, __nv_bfloat16>) {
                long long row = null_row;
                if (idx != nullptr) row = idx[b] < 0 ? 0 : (idx[b] > max_row ? max_row : idx[b]);  // never read outside the table
                if (row >= 0) v += table[static_cast<size_t>(row) * N + j];
                out[static_cast<size_t>(b) * N + j] = __float2bfloat16(silu(v));
            } else {
                out[static_cast<size_t>(b) * N + j] = silu(v);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// K1: patch embed (timm PatchEmbed conv k=p, s=p as a 16-wide dot product) + bias + pos_embed -> fp32 tokens.
// x is NCHW fp32 with x_rows samples; network row b reads sample (b % x_rows) (CFG duplicates the latents,
// reference models/DiT.py:279-280).  p = 2, C = 4 => patch vector (c, p, q) of 16 floats.
// One block = 8 tokens; thread d handles features d, d+256, ...
__global__ void __launch_bounds__(256)
patch_embed_kernel(const float* __restrict__ x, int x_rows, const float* __restrict__ Wt /*[16,D] (transposed at upload)*/,
                   const float* __restrict__ bias, const float* __restrict__ pos /*[T,D]*/, float* __restrict__ tok,
                   int D, int G /*grid side*/, int C, int M) {
    __shared__ float patch[8][16];
    const int T = G * G, HW = 2 * G;
    const int m0 = blockIdx.x * 8;
    if (threadIdx.x < 128) {
        const int tk = threadIdx.x >> 4, e = threadIdx.x & 15;
        const int m = m0 + tk;
        float v = 0.f;
        if (m < M) {
            const int b = (m / T) % x_rows, t = m % T;
            const int gh = t / G, gw = t % G;
            const int c = e >> 2, p = (e >> 1) & 1, q = e & 1;
            v = x[((static_cast<size_t>(b) * C + c) * HW + (2 * gh + p)) * HW + 2 * gw + q];
        }
        patch[tk][e] = v;
    }
    __syncthreads();
    // thread = 4 consecutive features (float4 stores, 512 B per warp); the 4 x 16 weights stay in registers
    for (int d4 = threadIdx.x; d4 < D / 4; d4 += 256) {
        float w[4][16];
#pragma unroll
        for (int e = 0; e < 16; ++e) {  // coalesced: consecutive threads read consecutive float4 of row e
            const float4 w4 = __ldg(reinterpret_cast<const float4*>(Wt + static_cast<size_t>(e) * D) + d4);
            w[0][e] = w4.x, w[1][e] = w4.y, w[2][e] = w4.z, w[3][e] = w4.w;
        }
        const float4 b4 = __ldg(reinterpret_cast<const float4*>(bias) + d4);
#pragma unroll
        for (int tk = 0; tk < 8; ++tk) {
            const int m = m0 + tk;
            if (m < M) {
                float a0 = b4.x, a1 = b4.y, a2 = b4.z, a3 = b4.w;
#pragma unroll
                for (int e = 0; e < 16; ++e) {
                    const float pe = patch[tk][e];
                    a0 = fmaf(w[0][e], pe, a0);
                    a1 = fmaf(w[1][e], pe, a1);
                    a2 = fmaf(w[2][e], pe, a2);
                    a3 = fmaf(w[3][e], pe, a3);
                }
                const float4 p4 = __ldg(reinterpret_cast<const float4*>(pos + static_cast<size_t>(m % T) * D) + d4);
                reinterpret_cast<float4*>(tok + static_cast<size_t>(m) * D)[d4] =
                    make_float4(a0 + p4.x, a1 + p4.y, a2 + p4.z, a3 + p4.w);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// K5/K9: LayerNorm (no affine, eps 1e-6) + adaLN modulate, fp32 tokens -> bf16 GEMM operand.
//   y = (x - mean) * rstd * (1 + scale[b]) + shift[b]        (reference models/DiT.py:20-21,119,121,129-130)
// HBM-bound (reads 4 B, writes 2 B per element).  Persistent blocks of 16 warps.  The token rows stream through a
// shared-memory ring filled by 1-D bulk async copies (cp.async.bulk + mbarrier transaction bytes): a stage holds a tile of
// 16 rows, one per warp, followed by the shift and scale vectors of the tile's sample, so loads of later tiles are in flight
// while the warps normalise the current one.  One warp per row, two-pass statistics in registers, coalesced bf16 stores.
// The per-row chain (shared-memory reads -> two warp reductions -> rsqrt -> modulate -> store, ~1500 clk with its waits) is
// latency-bound, so 16 rows in flight per SM hide more of it (tests/tools/l2_residency.cu times the pass with x in L2 and
// after a flush).
// Tiles are dealt round-robin, so the whole grid sweeps M upwards (down = 0) or downwards (down = 1) in time: a sweep that
// starts where the producer of x finished finds those rows still in L2.
// rows_per_sample must be a multiple of 16 (launch_ln checks it), so a tile never straddles two samples.
// OutT = __nv_fp8_e4m3 (the DiT's FP8 mode): the modulated row stays in registers, one more warp reduction takes its amax, and
// the row is written as e4m3 codes y = v / ys[row] with ys[row] = e4m3_row_scale(amax) (the A operand of the FP8 GEMM).
constexpr int kLnRows = 16;
__host__ __device__ constexpr int ln_stages(int NV) { return NV > 8 ? 2 : 3; }  // 3 x 72 KB at D = 1024
// dynamic shared memory of ln_modulate_kernel<NV>: per stage kLnRows rows of x, then the shift and scale vectors
__host__ __device__ constexpr int ln_smem_bytes(int NV) { return ln_stages(NV) * (kLnRows + 2) * NV * 128 * 4; }

LFM_DEVICE void bulk_load_1d(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(reinterpret_cast<uint64_t>(gsrc)), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

template <int NV, typename OutT = __nv_bfloat16>  // NV = D / 128 float4 per lane
__global__ void __launch_bounds__(kLnRows * 32, 1)
ln_modulate_kernel(const float* __restrict__ x, OutT* __restrict__ y, const float* __restrict__ shift,
                   const float* __restrict__ scale, int mod_stride, int rows_per_sample, int M, int down,
                   float* __restrict__ ys /* FP8 only: [M] row scales */) {
    constexpr int D = NV * 128;
    constexpr int kLnStages = ln_stages(NV);
    constexpr uint32_t kStageBytes = (kLnRows + 2) * D * 4;
    extern __shared__ __align__(128) uint8_t ln_smem[];
    __shared__ __align__(8) uint64_t full_bar[kLnStages];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int num_tiles = (M + kLnRows - 1) / kLnRows;
    const int my_tiles = (num_tiles - static_cast<int>(blockIdx.x) + static_cast<int>(gridDim.x) - 1) / static_cast<int>(gridDim.x);
    auto tile_of = [&](int i) {
        const int g = static_cast<int>(blockIdx.x) + i * static_cast<int>(gridDim.x);
        return down ? num_tiles - 1 - g : g;
    };
    if (threadIdx.x == 0) {
        for (int s = 0; s < kLnStages; ++s) mbar_init(&full_bar[s], 1);
        fence_barrier_init();
        fence_proxy_async();
    }
    __syncthreads();
    pdl_wait();
    pdl_trigger();
    auto issue = [&](int i) {  // thread 0: load tile tile_of(i) and its sample's modulation vectors into stage i % kLnStages
        const int tile = tile_of(i);
        const int rows = min(kLnRows, M - tile * kLnRows);
        const uint32_t bytes = static_cast<uint32_t>(rows) * D * 4;
        uint8_t* stage = ln_smem + (i % kLnStages) * kStageBytes;
        uint64_t* bar = &full_bar[i % kLnStages];
        mbar_arrive_expect_tx(bar, bytes + 2u * D * 4);
        const size_t boff = static_cast<size_t>(tile * kLnRows / rows_per_sample) * mod_stride;
        bulk_load_1d(stage + kLnRows * D * 4, shift + boff, D * 4, bar);
        bulk_load_1d(stage + (kLnRows + 1) * D * 4, scale + boff, D * 4, bar);
        bulk_load_1d(stage, x + static_cast<size_t>(tile) * kLnRows * D, bytes, bar);
    };
    if (threadIdx.x == 0)
        for (int i = 0; i < kLnStages && i < my_tiles; ++i) issue(i);

    for (int i = 0; i < my_tiles; ++i) {
        const int stage = i % kLnStages;
        const uint32_t parity = (i / kLnStages) & 1;
        const int row = tile_of(i) * kLnRows + warp;
        mbar_wait(&full_bar[stage], parity);
        if (row < M) {
            const float4* xp = reinterpret_cast<const float4*>(ln_smem + stage * kStageBytes + warp * D * 4);
            float4 v[NV];
            float s = 0.f;
#pragma unroll
            for (int m = 0; m < NV; ++m) {
                v[m] = xp[m * 32 + lane];
                s += (v[m].x + v[m].y) + (v[m].z + v[m].w);
            }
            const float mean = warp_sum(s) / static_cast<float>(D);
            float ss = 0.f;
#pragma unroll
            for (int m = 0; m < NV; ++m) {
                const float a = v[m].x - mean, b = v[m].y - mean, c = v[m].z - mean, d = v[m].w - mean;
                ss += (a * a + b * b) + (c * c + d * d);
            }
            const float rstd = rsqrtf(warp_sum(ss) / static_cast<float>(D) + 1e-6f);
            const float4* shs = reinterpret_cast<const float4*>(ln_smem + stage * kStageBytes + kLnRows * D * 4);
            if constexpr (std::is_same_v<OutT, __nv_fp8_e4m3>) {
                float amax = 0.f;
#pragma unroll
                for (int m = 0; m < NV; ++m) {
                    const float4 sh = shs[m * 32 + lane], sc = shs[D / 4 + m * 32 + lane];
                    v[m].x = fmaf((v[m].x - mean) * rstd, 1.f + sc.x, sh.x);
                    v[m].y = fmaf((v[m].y - mean) * rstd, 1.f + sc.y, sh.y);
                    v[m].z = fmaf((v[m].z - mean) * rstd, 1.f + sc.z, sh.z);
                    v[m].w = fmaf((v[m].w - mean) * rstd, 1.f + sc.w, sh.w);
                    amax = fmaxf(amax, fmaxf(fmaxf(fabsf(v[m].x), fabsf(v[m].y)), fmaxf(fabsf(v[m].z), fabsf(v[m].w))));
                }
                const float s_row = e4m3_row_scale(warp_max(amax));
                uint32_t* yp = reinterpret_cast<uint32_t*>(y + static_cast<size_t>(row) * D);
#pragma unroll
                for (int m = 0; m < NV; ++m)
                    yp[m * 32 + lane] = pack_e4m3x4(__fdiv_rn(v[m].x, s_row), __fdiv_rn(v[m].y, s_row), __fdiv_rn(v[m].z, s_row),
                                                    __fdiv_rn(v[m].w, s_row));
                if (lane == 0) ys[row] = s_row;
            } else {
                uint2* yp = reinterpret_cast<uint2*>(y + static_cast<size_t>(row) * D);
#pragma unroll
                for (int m = 0; m < NV; ++m) {
                    const float4 sh = shs[m * 32 + lane], sc = shs[D / 4 + m * 32 + lane];
                    const float a = fmaf((v[m].x - mean) * rstd, 1.f + sc.x, sh.x);
                    const float b = fmaf((v[m].y - mean) * rstd, 1.f + sc.y, sh.y);
                    const float c = fmaf((v[m].z - mean) * rstd, 1.f + sc.z, sh.z);
                    const float d = fmaf((v[m].w - mean) * rstd, 1.f + sc.w, sh.w);
                    yp[m * 32 + lane] = make_uint2(pack_bf16x2(a, b), pack_bf16x2(c, d));
                }
            }
        }
        __syncthreads();  // every warp has consumed this stage
        if (threadIdx.x == 0 && i + kLnStages < my_tiles) issue(i + kLnStages);
    }
}

// ------------------------------------------------------------------------------------------------
// K11: FinalLayer (LN + modulate + Linear(D, p*p*C)) + unpatchify, fp32 (reference models/DiT.py:134-149,230-243).
// Out-feature order of the linear is (p, q, c) -> pixel (c, 2h+p, 2w+q).  One warp per token; the 16 x D weight
// sits in shared memory.  Writes v_net[b, c, :, :] (NCHW fp32).
__global__ void __launch_bounds__(256)
final_layer_kernel(const float* __restrict__ x, const float* __restrict__ shift, const float* __restrict__ scale,
                   int mod_stride, const float* __restrict__ W /*[16, D]*/, const float* __restrict__ bias,
                   float* __restrict__ v_net, int M, int D, int G, int C) {
    extern __shared__ float sW[];  // [16][D]
    constexpr int MAXV = 12;
    const int P = 4 * C;  // p*p*C outputs (p = 2)
    for (int i = threadIdx.x; i < P * D / 4; i += blockDim.x)
        reinterpret_cast<float4*>(sW)[i] = __ldg(reinterpret_cast<const float4*>(W) + i);
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nv = D / 128, T = G * G, HW = 2 * G;
    for (int row = blockIdx.x * 8 + warp; row < M; row += gridDim.x * 8) {
        const float4* xp = reinterpret_cast<const float4*>(x + static_cast<size_t>(row) * D);
        float4 v[MAXV];
        float s = 0.f;
#pragma unroll
        for (int m = 0; m < MAXV; ++m)
            if (m < nv) {
                v[m] = xp[m * 32 + lane];
                s += (v[m].x + v[m].y) + (v[m].z + v[m].w);
            }
        const float mean = warp_sum(s) / static_cast<float>(D);
        float ss = 0.f;
#pragma unroll
        for (int m = 0; m < MAXV; ++m)
            if (m < nv) {
                const float a = v[m].x - mean, b = v[m].y - mean, c = v[m].z - mean, d = v[m].w - mean;
                ss += (a * a + b * b) + (c * c + d * d);
            }
        const float rstd = rsqrtf(warp_sum(ss) / static_cast<float>(D) + 1e-6f);
        const int bidx = row / T, t = row % T;
        const size_t boff = static_cast<size_t>(bidx) * mod_stride;
        const float4* shp = reinterpret_cast<const float4*>(shift + boff);
        const float4* scp = reinterpret_cast<const float4*>(scale + boff);
#pragma unroll
        for (int m = 0; m < MAXV; ++m)
            if (m < nv) {
                const float4 sh = __ldg(shp + m * 32 + lane), sc = __ldg(scp + m * 32 + lane);
                v[m].x = fmaf((v[m].x - mean) * rstd, 1.f + sc.x, sh.x);
                v[m].y = fmaf((v[m].y - mean) * rstd, 1.f + sc.y, sh.y);
                v[m].z = fmaf((v[m].z - mean) * rstd, 1.f + sc.z, sh.z);
                v[m].w = fmaf((v[m].w - mean) * rstd, 1.f + sc.w, sh.w);
            }
        const int gh = t / G, gw = t % G;
        // 16 dot products: per-lane partial sums, then a butterfly that halves the number of live values per step
        // (8 + 4 + 2 + 1 + 1 = 16 shuffles instead of 16 x 5): lane l ends up with output j = (l >> 1) & 15.
        float part[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            const float4* wp = reinterpret_cast<const float4*>(sW + static_cast<size_t>(j) * D);
            float acc = 0.f;
#pragma unroll
            for (int m = 0; m < MAXV; ++m)
                if (m < nv) {
                    const float4 w4 = wp[m * 32 + lane];
                    acc = fmaf(w4.x, v[m].x, acc);
                    acc = fmaf(w4.y, v[m].y, acc);
                    acc = fmaf(w4.z, v[m].z, acc);
                    acc = fmaf(w4.w, v[m].w, acc);
                }
            part[j] = acc;
        }
        {
            const bool hi = lane & 16;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const float send = hi ? part[i] : part[i + 8];
                const float keep = hi ? part[i + 8] : part[i];
                part[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
            }
        }
        {
            const bool hi = lane & 8;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float send = hi ? part[i] : part[i + 4];
                const float keep = hi ? part[i + 4] : part[i];
                part[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
            }
        }
        {
            const bool hi = lane & 4;
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const float send = hi ? part[i] : part[i + 2];
                const float keep = hi ? part[i + 2] : part[i];
                part[i] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
            }
        }
        {
            const bool hi = lane & 2;
            const float send = hi ? part[0] : part[1];
            const float keep = hi ? part[1] : part[0];
            part[0] = keep + __shfl_xor_sync(0xffffffffu, send, 2);
        }
        part[0] += __shfl_xor_sync(0xffffffffu, part[0], 1);
        if ((lane & 1) == 0) {
            // output index owned by this lane: bit4 -> +8, bit3 -> +4, bit2 -> +2, bit1 -> +1
            const int j = ((lane >> 4) & 1) * 8 + ((lane >> 3) & 1) * 4 + ((lane >> 2) & 1) * 2 + ((lane >> 1) & 1);
            const int p = j / (2 * C), q = (j / C) & 1, c = j % C;
            v_net[((static_cast<size_t>(bidx) * C + c) * HW + (2 * gh + p)) * HW + 2 * gw + q] = part[0] + bias[j];
        }
    }
}

// ------------------------------------------------------------------------------------------------
// K12: classifier-free-guidance combine (reference models/DiT.py:285-290): rows [0,n) conditional, [n,2n) null.
//   g = u + s (c - u).   dup != 0 also writes g into the second half (the reference returns cat[g, g]).
__global__ void cfg_combine_kernel(const float* __restrict__ v_net, float* __restrict__ out, size_t n_half, float s,
                                   int dup) {
    const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n_half) return;
    const float c = v_net[i], u = v_net[i + n_half];
    const float g = u + s * (c - u);
    out[i] = g;
    if (dup) out[i + n_half] = g;
}

// ------------------------------------------------------------------------------------------------
// K13: fixed-step solver updates.  The nodes t_grid, a table of every step's S stage times (S = 1 Euler, 2 Heun and
// midpoint, 4 rk4; built and perturbed on the host) and the step index live in device memory, so one captured CUDA
// graph serves every step of a trajectory with no host involvement.  The update kernels read dt = t[i+1] - t[i] from
// the nodes at the counter; step_advance_kernel, the last kernel of a step graph, bumps it.
struct StepState {
    int step;  // current interval index i
};

// t_eval[0..S) = the stage times of interval `step`: t_stage[step * S + j]
__global__ void stage_time_kernel(const float* __restrict__ t_stage, const StepState* __restrict__ st, int S,
                                  float* __restrict__ t_eval) {
    if (blockIdx.x == 0 && static_cast<int>(threadIdx.x) < S) t_eval[threadIdx.x] = t_stage[st->step * S + threadIdx.x];
}

// Euler:  x <- x + v * (sign * (t[i+1] - t[i]))      (karras_sample.py:116-117; torchdiffeq y0 + dt*f with the
// reversed-time sign folded in: there dt = s[i+1]-s[i] = -(t[i+1]-t[i]) and f = -v, the same product)
__global__ void euler_update_kernel(float* __restrict__ x, const float* __restrict__ v, const float* __restrict__ t_grid,
                                    const StepState* __restrict__ st, size_t n) {
    const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float dt = t_grid[st->step + 1] - t_grid[st->step];
    x[i] = x[i] + v[i] * dt;
}

// Heun predictor: x_pred = x + dt * d_cur (x itself is kept)     (karras_sample.py:152)
__global__ void heun_predict_kernel(const float* __restrict__ x, const float* __restrict__ d_cur,
                                    float* __restrict__ x_pred, const float* __restrict__ t_grid,
                                    const StepState* __restrict__ st, size_t n) {
    const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float dt = t_grid[st->step + 1] - t_grid[st->step];
    x_pred[i] = x[i] + dt * d_cur[i];
}

// Heun corrector: x <- x + dt * (0.5 d_cur + 0.5 d_prime)     (karras_sample.py:155-159; the intervals past the
// reference's corrector guard replay an Euler step instead)
__global__ void heun_correct_kernel(float* __restrict__ x, const float* __restrict__ d_cur,
                                    const float* __restrict__ d_prime, const float* __restrict__ t_grid,
                                    const StepState* __restrict__ st, size_t n) {
    const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int step = st->step;
    const float dt = t_grid[step + 1] - t_grid[step];
    x[i] = x[i] + dt * (0.5f * d_cur[i] + 0.5f * d_prime[i]);
}

__global__ void step_advance_kernel(StepState* st) {
    if (threadIdx.x == 0 && blockIdx.x == 0) st->step += 1;
}

// ------------------------------------------------------------------------------------------------
// K14: dopri5 arithmetic (torchdiffeq rk_common; SURVEY 8(c)).  k[j] are the 7 stage derivatives.
struct RkPtrs {
    const float* k[7];
};
struct RkCoef {   // passed by value as a kernel argument: no device upload, no host synchronisation
    float c[8];
};
__global__ void set_scalar_kernel(float* dst, float v) {
    if (threadIdx.x == 0 && blockIdx.x == 0) dst[0] = v;
}

// One attempted dopri5 step's numbers, uploaded once per step (the captured step graph reads them from device memory):
// stage i forms y0 + sum_j coef[i][j] k_j (coefficients already multiplied by dt) and evaluates the network at t[i].
struct DpStep {
    float coef[6][8];
    float t[8];      // model time of the 6 stage evaluations (t = -s)
    float cerr[8];   // dt * c_err
};
__global__ void rk_combine_dev_kernel(const float* __restrict__ y0, RkPtrs kp, int nk, const float* __restrict__ coef,
                                      float* __restrict__ y_out, size_t n) {
    const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float acc = 0.f;
    for (int j = 0; j < nk; ++j) acc = fmaf(kp.k[j][i], coef[j], acc);
    y_out[i] = y0[i] + acc;
}
// accepted step: y0 <- y1, f0 <- k7 (FSAL) as copies, so that the captured graph keeps its buffer pointers
__global__ void dp_accept_kernel(float* __restrict__ y0, const float* __restrict__ y1, float* __restrict__ k0,
                                 const float* __restrict__ k6, size_t n) {
    const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    y0[i] = y1[i];
    k0[i] = k6[i];
}

// partial[blk] = sum over this block's elements of ((a - b) / (atol + rtol * max(|y0|, |y1|)))^2
// a == nullptr: a = sum_j coef[j] * k[j] (the embedded error estimate).  b may be nullptr.  Warp-shuffle reduce.
constexpr int kRmsBlocks = 128;
__global__ void __launch_bounds__(256)
rms_ratio_partial_kernel(const float* __restrict__ a, const float* __restrict__ b, RkPtrs kp,
                         RkCoef coef, const float* __restrict__ y0, const float* __restrict__ y1,
                         float atol, float rtol, size_t n, double* __restrict__ partial,
                         const float* __restrict__ coef_dev = nullptr /* overrides coef (captured step graph) */) {
    if (coef_dev != nullptr)
        for (int j = 0; j < 7; ++j) coef.c[j] = coef_dev[j];
    __shared__ double wsum[8];
    double acc = 0.0;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
         i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        float num;
        if (a != nullptr) {
            num = a[i] - (b != nullptr ? b[i] : 0.f);
        } else {
            num = 0.f;
            for (int j = 0; j < 7; ++j) num = fmaf(kp.k[j][i], coef.c[j], num);
        }
        const float tol = atol + rtol * fmaxf(fabsf(y0[i]), fabsf(y1[i]));
        const float r = num / tol;
        acc += static_cast<double>(r) * static_cast<double>(r);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < 8; ++w) t += wsum[w];
        partial[blockIdx.x] = t;
    }
}
// out[0] = sqrt(sum(partial) / n)   (fixed summation order => deterministic)
__global__ void rms_finalize_kernel(const double* __restrict__ partial, int nblk, size_t n, float* __restrict__ out) {
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        double t = 0.0;
        for (int i = 0; i < nblk; ++i) t += partial[i];
        out[0] = static_cast<float>(sqrt(t / static_cast<double>(n)));
    }
}

// dense-output quartic of the last accepted step evaluated at x in [0,1] (torchdiffeq _interp_fit/_interp_evaluate)
__global__ void dopri_interp_kernel(const float* __restrict__ y0, const float* __restrict__ y1, RkPtrs kp,
                                    RkCoef coef_mid /*dt * c_mid*/, float dt, float xq,
                                    float* __restrict__ out, size_t n) {
    const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float mid = 0.f;
    for (int j = 0; j < 7; ++j) mid = fmaf(kp.k[j][i], coef_mid.c[j], mid);
    const float a0 = y0[i], a1 = y1[i], ym = a0 + mid, f0 = kp.k[0][i], f1 = kp.k[6][i];
    const float ca = 2.f * dt * (f1 - f0) - 8.f * (a1 + a0) + 16.f * ym;
    const float cb = dt * (5.f * f0 - 3.f * f1) + 18.f * a0 + 14.f * a1 - 32.f * ym;
    const float cc = dt * (f1 - 4.f * f0) - 11.f * a0 - 5.f * a1 + 16.f * ym;
    const float cd = dt * f0;
    float total = a0 + xq * cd;
    float xp = xq * xq;
    total += xp * cc;
    xp *= xq;
    total += xp * cb;
    xp *= xq;
    total += xp * ca;
    out[i] = total;
}

// torchdiffeq fixed-grid midpoint / rk4 (3/8 rule, rk4_alt_step_func) stage arithmetic, written in the same
// operation order as the Python expressions (real-time form: dt = t1 - t0 read from the nodes at the step counter, k = v).
//   mode 0: out = y0 + k1 * h                        (midpoint: h = 0.5 dt)
//   mode 1: out = y0 + dt * k2                       (midpoint result)
//   mode 2: out = y0 + (dt * k1) * (1/3)
//   mode 3: out = y0 + dt * (k2 - k1 * (1/3))
//   mode 4: out = y0 + dt * ((k1 - k2) + k3)
//   mode 5: out = y0 + ((k1 + 3 (k2 + k3)) + k4) * dt * 0.125
__global__ void fixed_rk_stage_kernel(int mode, const float* y0 /*may alias out*/, const float* __restrict__ k1,
                                      const float* __restrict__ k2, const float* __restrict__ k3,
                                      const float* __restrict__ k4, const float* __restrict__ t_grid,
                                      const StepState* __restrict__ st, float* out, size_t n) {
    const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float dt = t_grid[st->step + 1] - t_grid[st->step];
    const float third = static_cast<float>(1.0 / 3.0);
    float r;
    switch (mode) {
        case 0: r = __fadd_rn(y0[i], __fmul_rn(k1[i], __fmul_rn(0.5f, dt))); break;
        case 1: r = __fadd_rn(y0[i], __fmul_rn(dt, k2[i])); break;
        case 2: r = __fadd_rn(y0[i], __fmul_rn(__fmul_rn(dt, k1[i]), third)); break;
        case 3: r = __fadd_rn(y0[i], __fmul_rn(dt, __fsub_rn(k2[i], __fmul_rn(k1[i], third)))); break;
        case 4: r = __fadd_rn(y0[i], __fmul_rn(dt, __fadd_rn(__fsub_rn(k1[i], k2[i]), k3[i]))); break;
        default:
            r = __fadd_rn(y0[i], __fmul_rn(__fmul_rn(__fadd_rn(__fadd_rn(k1[i], __fmul_rn(3.0f, __fadd_rn(k2[i], k3[i]))), k4[i]), dt), 0.125f));
            break;
    }
    out[i] = r;
}

__global__ void axpy_kernel(const float* __restrict__ y, const float* __restrict__ f, float h, float* __restrict__ out,
                            size_t n) {
    const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < n) out[i] = y[i] + h * f[i];
}
__global__ void negate_kernel(float* __restrict__ v, size_t n) {
    const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < n) v[i] = -v[i];
}

// [rows, cols] fp32 -> [cols, rows] fp32 (patch-embed weight [D,16] -> [16,D])
__global__ void transpose_f32_kernel(const float* __restrict__ in, float* __restrict__ out, int rows, int cols) {
    const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= static_cast<size_t>(rows) * cols) return;
    const int r = static_cast<int>(i / cols), c = static_cast<int>(i % cols);
    out[static_cast<size_t>(c) * rows + r] = in[i];
}

// fp32 -> bf16 weight repack (nn.Linear weights are already [N, K] K-major: a plain cast)
__global__ void f32_to_bf16_kernel(const float* __restrict__ in, __nv_bfloat16* __restrict__ out, size_t n) {
    pdl_wait();  // PDL: nothing of the previous kernel's output is touched above this line
    pdl_trigger();
    const size_t i = (static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x) * 4;
    if (i + 3 < n) {
        const float4 v = *reinterpret_cast<const float4*>(in + i);
        *reinterpret_cast<uint2*>(out + i) = make_uint2(pack_bf16x2(v.x, v.y), pack_bf16x2(v.z, v.w));
    } else {
        for (size_t j = i; j < n; ++j) out[j] = __float2bfloat16(in[j]);
    }
}

// ------------------------------------------------------------------------------------------------
// DiT geometries other than (patch 2, 32 x 32 latents): patch sizes 4 / 8 and latent sides that give 16, 64 or 256 tokens
// (reference models/DiT.py:355-415 - the /4 and /8 entries of DiT_models; img_resolution = image_size // f).  Both ends of
// the network are < 0.1 % of its work, so these are plain kernels; the patch-2 / 32 x 32 presets keep the specialised ones.
//
// Patch embed for any p: patch vector (c, p, q) of P = C p^2 floats (timm PatchEmbed conv weight [D, C, p, p]), 8 tokens per block.
__global__ void __launch_bounds__(256)
patch_embed_generic_kernel(const float* __restrict__ x, int x_rows, const float* __restrict__ Wt /*[P, D]*/,
                           const float* __restrict__ bias, const float* __restrict__ pos /*[T, D]*/, float* __restrict__ tok,
                           int D, int G, int C, int p, int M) {
    extern __shared__ float patch_sm[];  // [8][P]
    const int P = C * p * p, T = G * G, HW = p * G;
    const int m0 = blockIdx.x * 8;
    for (int i = threadIdx.x; i < 8 * P; i += 256) {
        const int tk = i / P, e = i % P;
        const int m = m0 + tk;
        float v = 0.f;
        if (m < M) {
            const int b = (m / T) % x_rows, t = m % T;
            const int gh = t / G, gw = t % G;
            const int c = e / (p * p), pp = (e / p) % p, q = e % p;
            v = x[((static_cast<size_t>(b) * C + c) * HW + (p * gh + pp)) * HW + p * gw + q];
        }
        patch_sm[i] = v;
    }
    __syncthreads();
    for (int d4 = threadIdx.x; d4 < D / 4; d4 += 256) {
        const float4 b4 = __ldg(reinterpret_cast<const float4*>(bias) + d4);
        float4 acc[8];
#pragma unroll
        for (int tk = 0; tk < 8; ++tk) acc[tk] = b4;
        for (int e = 0; e < P; ++e) {
            const float4 w4 = __ldg(reinterpret_cast<const float4*>(Wt + static_cast<size_t>(e) * D) + d4);
#pragma unroll
            for (int tk = 0; tk < 8; ++tk) {
                const float pe = patch_sm[tk * P + e];
                acc[tk].x = fmaf(w4.x, pe, acc[tk].x);
                acc[tk].y = fmaf(w4.y, pe, acc[tk].y);
                acc[tk].z = fmaf(w4.z, pe, acc[tk].z);
                acc[tk].w = fmaf(w4.w, pe, acc[tk].w);
            }
        }
#pragma unroll
        for (int tk = 0; tk < 8; ++tk) {
            const int m = m0 + tk;
            if (m < M) {
                const float4 p4 = __ldg(reinterpret_cast<const float4*>(pos + static_cast<size_t>(m % T) * D) + d4);
                reinterpret_cast<float4*>(tok + static_cast<size_t>(m) * D)[d4] =
                    make_float4(acc[tk].x + p4.x, acc[tk].y + p4.y, acc[tk].z + p4.z, acc[tk].w + p4.w);
            }
        }
    }
}

// FinalLayer + unpatchify for any p: LN + modulate in registers (one warp per token), then the P_out = p p C dot products
// against the weight rows read through L2; out-feature j = (pp p + q) C + c  ->  pixel (c, p gh + pp, p gw + q).
__global__ void __launch_bounds__(256)
final_layer_generic_kernel(const float* __restrict__ x, const float* __restrict__ shift, const float* __restrict__ scale,
                           int mod_stride, const float* __restrict__ W /*[P_out, D]*/, const float* __restrict__ bias,
                           float* __restrict__ v_net, int M, int D, int G, int C, int p) {
    constexpr int MAXV = 12;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nv = D / 128, T = G * G, HW = p * G, Pout = p * p * C;
    for (int row = blockIdx.x * 8 + warp; row < M; row += gridDim.x * 8) {
        const float4* xp = reinterpret_cast<const float4*>(x + static_cast<size_t>(row) * D);
        float4 v[MAXV];
        float s = 0.f;
#pragma unroll
        for (int m = 0; m < MAXV; ++m)
            if (m < nv) {
                v[m] = xp[m * 32 + lane];
                s += (v[m].x + v[m].y) + (v[m].z + v[m].w);
            }
        const float mean = warp_sum(s) / static_cast<float>(D);
        float ss = 0.f;
#pragma unroll
        for (int m = 0; m < MAXV; ++m)
            if (m < nv) {
                const float a = v[m].x - mean, b = v[m].y - mean, c = v[m].z - mean, d = v[m].w - mean;
                ss += (a * a + b * b) + (c * c + d * d);
            }
        const float rstd = rsqrtf(warp_sum(ss) / static_cast<float>(D) + 1e-6f);
        const int bidx = row / T, t = row % T;
        const size_t boff = static_cast<size_t>(bidx) * mod_stride;
        const float4* shp = reinterpret_cast<const float4*>(shift + boff);
        const float4* scp = reinterpret_cast<const float4*>(scale + boff);
#pragma unroll
        for (int m = 0; m < MAXV; ++m)
            if (m < nv) {
                const float4 sh = __ldg(shp + m * 32 + lane), sc = __ldg(scp + m * 32 + lane);
                v[m].x = fmaf((v[m].x - mean) * rstd, 1.f + sc.x, sh.x);
                v[m].y = fmaf((v[m].y - mean) * rstd, 1.f + sc.y, sh.y);
                v[m].z = fmaf((v[m].z - mean) * rstd, 1.f + sc.z, sh.z);
                v[m].w = fmaf((v[m].w - mean) * rstd, 1.f + sc.w, sh.w);
            }
        const int gh = t / G, gw = t % G;
        for (int j0 = 0; j0 < Pout; j0 += 32) {
            float mine = 0.f;
            for (int jj = 0; jj < 32 && j0 + jj < Pout; ++jj) {
                const float4* wp = reinterpret_cast<const float4*>(W + static_cast<size_t>(j0 + jj) * D);
                float acc = 0.f;
#pragma unroll
                for (int m = 0; m < MAXV; ++m)
                    if (m < nv) {
                        const float4 w4 = __ldg(wp + m * 32 + lane);
                        acc = fmaf(w4.x, v[m].x, acc);
                        acc = fmaf(w4.y, v[m].y, acc);
                        acc = fmaf(w4.z, v[m].z, acc);
                        acc = fmaf(w4.w, v[m].w, acc);
                    }
                acc = warp_sum(acc);
                if (lane == jj) mine = acc;
            }
            const int j = j0 + lane;
            if (j < Pout) {
                const int pp = j / (p * C), q = (j / C) % p, c = j % C;
                v_net[((static_cast<size_t>(bidx) * C + c) * HW + (p * gh + pp)) * HW + p * gw + q] = mine + bias[j];
            }
        }
    }
}

// Orders of the 3 C qkv rows (C = heads * dh; which = q, k, v).  The first two are also the layouts of lfm_dbg_attention
// (LFM_QKV_TIMM, LFM_QKV_HEAD_MAJOR).
//   QKV_TIMM        which * C + head * dh + c      timm's Attention (models/DiT.py:120 / SURVEY D6): the DiT checkpoints
//   QKV_HEAD_MAJOR  head * 3 dhp + which * dhp + c  what the mma.sync and SIMT attention kernels read; dhp >= dh is the stored
//                                                   head width, rows c >= dh are zero (DiT-XL's 72 channels padded to 80, so
//                                                   q.k^T and P.V are unchanged and the padded output channels are exactly zero)
//   QKV_EDM         head * 3 dh + c * 3 + which     UNetBlock.qkv (EDM.py:277-281), a checkpoint order only
enum QkvOrder { QKV_TIMM = 0, QKV_HEAD_MAJOR = 1, QKV_EDM = 2 };

// The source row of destination row r when the qkv rows are re-ordered ONCE at upload from order `src` to order `dst`
// (dhp = dh unless dst is QKV_HEAD_MAJOR); -1: a zero padding row.
LFM_DEVICE int qkv_src_row(int r, int heads, int dh, int dhp, int src, int dst) {
    int h, which, c;
    if (dst == QKV_TIMM) {
        which = r / (heads * dh), h = (r / dh) % heads, c = r % dh;
    } else {
        h = r / (3 * dhp), which = (r % (3 * dhp)) / dhp, c = r % dhp;
        if (c >= dh) return -1;
    }
    return src == QKV_EDM ? h * 3 * dh + c * 3 + which : which * heads * dh + h * dh + c;
}
// weight [3 C, K] fp32 -> [3 heads dhp, K] bf16, or fp32 (the source of the FP8 mode's quantisation)
template <typename OutT>
__global__ void qkv_weight_reorder_kernel(const float* __restrict__ w, OutT* __restrict__ out, int K, int heads, int dh, int dhp,
                                          int src, int dst) {
    const size_t n = static_cast<size_t>(3) * heads * dhp * K;
    const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int r = qkv_src_row(static_cast<int>(i / K), heads, dh, dhp, src, dst);
    out[i] = static_cast<OutT>(r >= 0 ? w[static_cast<size_t>(r) * K + i % K] : 0.f);
}
// Per-row e4m3 quantisation of an fp32 weight [N, K] (the FP8 mode's qkv and fc1): scales[n] = e4m3_row_scale(amax |w[n, :]|),
// codes[n, k] = e4m3(w[n, k] / scales[n]).  One warp per row; zero rows (DiT-XL's padded head channels) get scale 1 and codes 0.
__global__ void quantize_rows_e4m3_kernel(const float* __restrict__ w, __nv_fp8_e4m3* __restrict__ codes, float* __restrict__ scales,
                                          int N, int K) {
    const int row = blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= N) return;
    const float* wr = w + static_cast<size_t>(row) * K;
    float amax = 0.f;
    for (int k = lane; k < K; k += 32) amax = fmaxf(amax, fabsf(wr[k]));
    const float s = e4m3_row_scale(warp_max(amax));
    uint8_t* cr = reinterpret_cast<uint8_t*>(codes) + static_cast<size_t>(row) * K;
    for (int k = lane; k < K; k += 32) cr[k] = __nv_cvt_float_to_fp8(__fdiv_rn(wr[k], s), __NV_SATFINITE, __NV_E4M3);
    if (lane == 0) scales[row] = s;
}
// bias [3 C] -> [3 heads dhp], fp32
__global__ void qkv_bias_reorder_kernel(const float* __restrict__ b, float* __restrict__ out, int heads, int dh, int dhp, int src, int dst) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 3 * heads * dhp) return;
    const int r = qkv_src_row(i, heads, dh, dhp, src, dst);
    out[i] = r >= 0 ? b[r] : 0.f;
}
// proj weight [D, D] -> [D, heads * dhp]: input feature head * dh + d moves to column head * dhp + d, zero columns for the padding
__global__ void dit_proj_weight_pad_kernel(const float* __restrict__ w, __nv_bfloat16* __restrict__ out, int D, int dh, int dhp) {
    const int Dq = D / dh * dhp;
    const size_t n = static_cast<size_t>(D) * Dq;
    const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int r = static_cast<int>(i / Dq), c = static_cast<int>(i % Dq);
    const int h = c / dhp, d = c % dhp;
    out[i] = d < dh ? __float2bfloat16(w[static_cast<size_t>(r) * D + h * dh + d]) : __float2bfloat16(0.f);
}

}  // namespace lfm
