// lfm_b200 - the non-GEMM kernels of the DiT velocity network and the ODE-solver arithmetic.
// All HBM- or latency-bound; plain CUDA cores, vectorised, coalesced.  fp32 everywhere except the bf16 tensors
// that feed the wgmma GEMMs.
#pragma once
#include "common.cuh"

namespace lfm {

// ------------------------------------------------------------------------------------------------
// K2: sinusoidal timestep features  tf[b, :] = [cos(t f_i) | sin(t f_i)], f_i = exp(-ln(1e4) i / 128)
// (reference models/DiT.py:43-62; raw t in [0,1], cos first).  t_numel == 1 broadcasts.
__global__ void timestep_features_kernel(const float* __restrict__ t, int t_numel, float* __restrict__ tf, int B) {
    const int b = blockIdx.x;
    const int i = threadIdx.x;  // 0..255
    if (b >= B) return;
    const float tv = t[t_numel == 1 ? 0 : b];
    const int k = i & 127;
    const float freq = expf(-9.210340371976184f * static_cast<float>(k) / 128.0f);
    const float a = tv * freq;
    tf[b * 256 + i] = (i < 128) ? cosf(a) : sinf(a);
}

// ------------------------------------------------------------------------------------------------
// K2/K3: skinny linear  out[b, j] = act( bias[j] + sum_k W[j, k] in[b, k] (+ table[idx[b], j]) )
// One warp per output feature j; the weight row stays in registers while the warp sweeps the batch.
// MODE 0: SiLU -> fp32 out          (t_embedder.mlp.0 + SiLU)
// MODE 1: + label-embedding row, then SiLU -> bf16 out (c = t_emb + y_emb; adaLN's leading SiLU, DiT.py:125,264)
template <int MODE>
__global__ void __launch_bounds__(256)
skinny_linear_kernel(const float* __restrict__ W, const float* __restrict__ bias, const float* __restrict__ in, int B,
                     int N, int K, const float* __restrict__ table, const long long* __restrict__ idx, int null_row,
                     float* __restrict__ out_f32, __nv_bfloat16* __restrict__ out_bf16) {
    constexpr int MAXV = 9;  // K <= 1152
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int j = blockIdx.x * 8 + warp;
    if (j >= N) return;
    const int nv = K / 128;  // float4 per lane
    float4 w[MAXV];
#pragma unroll
    for (int m = 0; m < MAXV; ++m)
        if (m < nv) w[m] = __ldg(reinterpret_cast<const float4*>(W + static_cast<size_t>(j) * K) + m * 32 + lane);
    const float bj = bias[j];
    for (int b = 0; b < B; ++b) {
        const float4* ip = reinterpret_cast<const float4*>(in + static_cast<size_t>(b) * K);
        float acc = 0.f;
#pragma unroll
        for (int m = 0; m < MAXV; ++m) {
            if (m < nv) {
                const float4 x = __ldg(ip + m * 32 + lane);
                acc = fmaf(w[m].x, x.x, acc);
                acc = fmaf(w[m].y, x.y, acc);
                acc = fmaf(w[m].z, x.z, acc);
                acc = fmaf(w[m].w, x.w, acc);
            }
        }
        acc = warp_sum(acc);
        if (lane == 0) {
            float v = acc + bj;
            if (MODE == 1) {
                long long row = (idx != nullptr) ? idx[b] : static_cast<long long>(null_row);
                row = row < 0 ? 0 : (row > null_row ? null_row : row);  // never read outside the table (null_row = last row)
                v += table[static_cast<size_t>(row) * N + j];
            }
            v = silu(v);
            if (MODE == 0)
                out_f32[static_cast<size_t>(b) * N + j] = v;
            else
                out_bf16[static_cast<size_t>(b) * N + j] = __float2bfloat16(v);
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
// HBM-bound (reads 4 B, writes 2 B per element).  Persistent blocks; the token rows stream through a 4-stage
// shared-memory ring filled by 1-D bulk async copies (cp.async.bulk + mbarrier transaction bytes), 8 rows per
// stage, so loads of later rows are always in flight while the 8 warps normalise the current ones.
// One warp per row, two-pass statistics in registers, coalesced bf16 stores.
// 16 warps, one row each per stage: the per-row chain (shared-memory reads -> two warp reductions -> rsqrt -> modulate -> store, ~1500
// clk with its waits) is latency-bound, so more rows in flight per SM hide more of it (tests/tools/l2_residency.cu times the pass with x
// in L2 and after a flush).
// Two shapes are kept for A/B runs (LFM_LN_ROWS = 8 | 16): 8 rows x 4 stages with per-warp modulation loads (round 1), and 16 rows x 3
// stages with the tile's shift / scale vectors staged next to its rows.
__host__ __device__ constexpr int ln_stages(int NV, int ROWS) { return ROWS == 8 ? 4 : (NV > 8 ? 2 : 3); }  // 16 rows: 3 x 72 KB at D = 1024

LFM_DEVICE void bulk_load_1d(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(reinterpret_cast<uint64_t>(gsrc)), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

LFM_DEVICE void bulk_load_1d_hint(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar, uint64_t policy) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(reinterpret_cast<uint64_t>(gsrc)), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
                 : "memory");
}

template <int NV, int kLnRows>  // NV = D / 128 float4 per lane; kLnRows = rows per stage = warps per block
__global__ void __launch_bounds__(kLnRows * 32, 1)
ln_modulate_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ y, const float* __restrict__ shift,
                   const float* __restrict__ scale, int mod_stride, int rows_per_sample, int M, int order_flags) {
    constexpr int D = NV * 128;
    constexpr int kLnStages = ln_stages(NV, kLnRows);
    const int order = order_flags & 3;          // tile order (below)
    const bool keep = (order_flags & 4) != 0;   // x is the residual stream: load with the evict_last L2 policy
    const uint64_t policy = keep ? l2_policy_evict_last() : 0;
    // a stage = kLnRows rows of x + the shift and scale vectors of the tile's sample: one copy of the two vectors per tile instead of
    // one per warp (8 KB per 4 KB row, twice the bytes of x through L2 -> SM).
    constexpr uint32_t kStageBytes = (kLnRows + (kLnRows == 16 ? 2 : 0)) * D * 4;
    const bool mod_smem = kLnRows == 16 && rows_per_sample % kLnRows == 0;  // a tile never straddles two samples
    extern __shared__ __align__(128) uint8_t ln_smem[];
    __shared__ __align__(8) uint64_t full_bar[kLnStages];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int num_tiles = (M + kLnRows - 1) / kLnRows;
    // order 0: contiguous tile range per block (keeps one block inside as few samples as possible);
    // order 1 / 2: tiles dealt round-robin so that the whole grid sweeps M upwards / downwards in time - a sweep that
    // starts where the producer of x finished finds those rows still in L2
    const int per = (num_tiles + gridDim.x - 1) / gridDim.x;
    const int t_begin = blockIdx.x * per;
    const int t_end = min(num_tiles, t_begin + per);
    const int my_tiles = order == 0 ? max(0, t_end - t_begin)
                                    : (num_tiles - static_cast<int>(blockIdx.x) + static_cast<int>(gridDim.x) - 1) / static_cast<int>(gridDim.x);
    auto tile_of = [&](int i) {
        if (order == 0) return t_begin + i;
        const int g = static_cast<int>(blockIdx.x) + i * static_cast<int>(gridDim.x);
        return order == 2 ? num_tiles - 1 - g : g;
    };
    if (threadIdx.x == 0) {
        for (int s = 0; s < kLnStages; ++s) mbar_init(&full_bar[s], 1);
        fence_barrier_init();
        fence_proxy_async();
    }
    __syncthreads();
    pdl_wait();
    pdl_trigger();
    auto issue = [&](int i) {  // thread 0: load tile t_begin + i into stage i % kLnStages
        const int tile = tile_of(i);
        const int rows = min(kLnRows, M - tile * kLnRows);
        const uint32_t bytes = static_cast<uint32_t>(rows) * D * 4;
        uint64_t* bar = &full_bar[i % kLnStages];
        mbar_arrive_expect_tx(bar, bytes + (mod_smem ? 2u * D * 4 : 0u));
        if (mod_smem) {
            const size_t boff = static_cast<size_t>(tile * kLnRows / rows_per_sample) * mod_stride;
            uint8_t* dst = ln_smem + (i % kLnStages) * kStageBytes + kLnRows * D * 4;
            bulk_load_1d(dst, shift + boff, D * 4, bar);
            bulk_load_1d(dst + D * 4, scale + boff, D * 4, bar);
        }
        if (keep)
            bulk_load_1d_hint(ln_smem + (i % kLnStages) * kStageBytes, x + static_cast<size_t>(tile) * kLnRows * D, bytes, bar, policy);
        else
            bulk_load_1d(ln_smem + (i % kLnStages) * kStageBytes, x + static_cast<size_t>(tile) * kLnRows * D, bytes, bar);
    };
    if (threadIdx.x == 0)
        for (int i = 0; i < kLnStages && i < my_tiles; ++i) issue(i);

    for (int i = 0; i < my_tiles; ++i) {
        const int stage = i % kLnStages;
        const uint32_t parity = (i / kLnStages) & 1;
        const int row = tile_of(i) * kLnRows + warp;
        const bool ok = row < M;
        // 8-row shape: the modulation vectors come from global memory, requested first so that their latency overlaps the wait
        float4 shr[kLnRows == 8 ? NV : 1], scr[kLnRows == 8 ? NV : 1];
        if (kLnRows == 8 && ok) {
            const size_t boff = static_cast<size_t>(row / rows_per_sample) * mod_stride;
            const float4* shp = reinterpret_cast<const float4*>(shift + boff);
            const float4* scp = reinterpret_cast<const float4*>(scale + boff);
#pragma unroll
            for (int m = 0; m < (kLnRows == 8 ? NV : 0); ++m) {
                shr[m] = __ldg(shp + m * 32 + lane);
                scr[m] = __ldg(scp + m * 32 + lane);
            }
        }
        mbar_wait(&full_bar[stage], parity);
        if (ok) {
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
            uint2* yp = reinterpret_cast<uint2*>(y + static_cast<size_t>(row) * D);
            const float4* shs = reinterpret_cast<const float4*>(ln_smem + stage * kStageBytes + kLnRows * D * 4);
            const size_t boff = static_cast<size_t>(row / rows_per_sample) * mod_stride;
            const float4* shg = reinterpret_cast<const float4*>(shift + boff);
            const float4* scg = reinterpret_cast<const float4*>(scale + boff);
#pragma unroll
            for (int m = 0; m < NV; ++m) {
                float4 sh, sc;
                if constexpr (kLnRows == 8) {
                    sh = shr[m], sc = scr[m];
                } else {
                    sh = mod_smem ? shs[m * 32 + lane] : __ldg(shg + m * 32 + lane);
                    sc = mod_smem ? shs[D / 4 + m * 32 + lane] : __ldg(scg + m * 32 + lane);
                }
                const float a = fmaf((v[m].x - mean) * rstd, 1.f + sc.x, sh.x);
                const float b = fmaf((v[m].y - mean) * rstd, 1.f + sc.y, sh.y);
                const float c = fmaf((v[m].z - mean) * rstd, 1.f + sc.z, sh.z);
                const float d = fmaf((v[m].w - mean) * rstd, 1.f + sc.w, sh.w);
                yp[m * 32 + lane] = make_uint2(pack_bf16x2(a, b), pack_bf16x2(c, d));
            }
        }
        __syncthreads();  // every warp has consumed this stage
        if (threadIdx.x == 0 && i + kLnStages < my_tiles) issue(i + kLnStages);
    }
}

// The same pass without the shared-memory ring (LFM_LN_ROWS=0): one row per warp straight from global memory into registers, 64
// registers so that 32 warps are resident per SM (8 independent row chains per scheduler instead of 4), the grid sweeping M in
// order (upwards, or downwards for order 2).  Same arithmetic in the same order as ln_modulate_kernel: identical results.
template <int NV, int THREADS = 256, int MINB = 4>
__global__ void __launch_bounds__(THREADS, MINB)
ln_modulate_direct_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ y, const float* __restrict__ shift,
                          const float* __restrict__ scale, int mod_stride, int rows_per_sample, int M, int order_flags) {
    // THREADS = 1024, MINB = 1 (LFM_LN_ROWS=32): the same 32 resident warps per SM as ONE persistent block per SM, which chains
    // through programmatic dependent launch like the ring version does.
    constexpr int D = NV * 128;
    constexpr int WARPS = THREADS / 32;
    pdl_wait();
    pdl_trigger();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const bool down = (order_flags & 3) == 2;
    for (int r = blockIdx.x * WARPS + warp; r < M; r += gridDim.x * WARPS) {
        const int row = down ? M - 1 - r : r;
        const float4* xp = reinterpret_cast<const float4*>(x + static_cast<size_t>(row) * D);
        const size_t boff = static_cast<size_t>(row / rows_per_sample) * mod_stride;
        const float4* shp = reinterpret_cast<const float4*>(shift + boff);
        const float4* scp = reinterpret_cast<const float4*>(scale + boff);
        uint2* yp = reinterpret_cast<uint2*>(y + static_cast<size_t>(row) * D);
        float4 v[NV];
#pragma unroll
        for (int m = 0; m < NV; ++m) v[m] = xp[m * 32 + lane];
        float s = 0.f;
#pragma unroll
        for (int m = 0; m < NV; ++m) s += (v[m].x + v[m].y) + (v[m].z + v[m].w);
        const float mean = warp_sum(s) / static_cast<float>(D);
        float ss = 0.f;
#pragma unroll
        for (int m = 0; m < NV; ++m) {
            const float a = v[m].x - mean, b = v[m].y - mean, c = v[m].z - mean, d = v[m].w - mean;
            ss += (a * a + b * b) + (c * c + d * d);
        }
        const float rstd = rsqrtf(warp_sum(ss) / static_cast<float>(D) + 1e-6f);
#pragma unroll
        for (int m = 0; m < NV; ++m) {
            const float4 sh = __ldg(shp + m * 32 + lane), sc = __ldg(scp + m * 32 + lane);
            const float a = fmaf((v[m].x - mean) * rstd, 1.f + sc.x, sh.x);
            const float b = fmaf((v[m].y - mean) * rstd, 1.f + sc.y, sh.y);
            const float c = fmaf((v[m].z - mean) * rstd, 1.f + sc.z, sh.z);
            const float d = fmaf((v[m].w - mean) * rstd, 1.f + sc.w, sh.w);
            yp[m * 32 + lane] = make_uint2(pack_bf16x2(a, b), pack_bf16x2(c, d));
        }
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
// K13: fixed-step solver updates.  The step schedule lives in device memory (t_grid) and the step index in
// a device counter, so one captured CUDA graph serves every step of a trajectory with no host involvement.
struct StepState {
    int step;         // current interval index i
    int n_intervals;  // len(t_grid) - 1
    int perturb;      // torchdiffeq options["perturb"]: the step's first evaluation sees t one fp32 ulp past the node
};

// Writes the model time(s) for the next evaluation: t_eval[0] = t_grid[step + which] (which: 0 = t_cur, 1 = t_next)
__global__ void step_time_kernel(const float* __restrict__ t_grid, const StepState* __restrict__ st, int which,
                                 float* __restrict__ t_eval) {
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        float t = t_grid[st->step + which];
        // Perturb.NEXT in torchdiffeq's negated time s = -t (nextafter(s, s + 1)) = one ulp DOWN in model time
        if (st->perturb && which == 0) t = nextafterf(t, t - 1.0f);
        t_eval[0] = t;
    }
}

// Euler:  x <- x + v * (sign * (t[i+1] - t[i]))      (karras_sample.py:116-117; torchdiffeq y0 + dt*f with the
// reversed-time sign folded in: there dt = s[i+1]-s[i] = -(t[i+1]-t[i]) and f = -v, the same product)
// advance != 0 bumps the device step counter (done by thread 0 of block 0 AFTER reading it - every block reads
// the counter before any block can finish, because the increment happens in a separate tiny kernel).
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

// Heun corrector: x <- x + dt * (0.5 d_cur + 0.5 d_prime) if step < corrector_limit else x <- x_pred
// (karras_sample.py:155-159; the guard `i < steps - 1` with the reference's never-overridden default steps = 40)
__global__ void heun_correct_kernel(float* __restrict__ x, const float* __restrict__ d_cur,
                                    const float* __restrict__ d_prime, const float* __restrict__ x_pred,
                                    const float* __restrict__ t_grid, const StepState* __restrict__ st,
                                    int corrector_limit, size_t n) {
    const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int step = st->step;
    if (step < corrector_limit) {
        const float dt = t_grid[step + 1] - t_grid[step];
        x[i] = x[i] + dt * (0.5f * d_cur[i] + 0.5f * d_prime[i]);
    } else {
        x[i] = x_pred[i];
    }
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

// y_out = y0 + sum_j (coef[j]) * k[j],  coef already multiplied by dt (fp32) on the host
__global__ void rk_combine_kernel(const float* __restrict__ y0, RkPtrs kp, int nk, RkCoef coef,
                                  float* __restrict__ y_out, size_t n) {
    const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float acc = 0.f;
    for (int j = 0; j < nk; ++j) acc = fmaf(kp.k[j][i], coef.c[j], acc);
    y_out[i] = y0[i] + acc;
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
// operation order as the Python expressions (real-time form: dt = t1 - t0, k = v).
//   mode 0: out = y0 + k1 * h                        (midpoint: h = 0.5 dt)
//   mode 1: out = y0 + dt * k2                       (midpoint result)
//   mode 2: out = y0 + (dt * k1) * (1/3)
//   mode 3: out = y0 + dt * (k2 - k1 * (1/3))
//   mode 4: out = y0 + dt * ((k1 - k2) + k3)
//   mode 5: out = y0 + ((k1 + 3 (k2 + k3)) + k4) * dt * 0.125
__global__ void fixed_rk_stage_kernel(int mode, const float* y0 /*may alias out*/, const float* __restrict__ k1,
                                      const float* __restrict__ k2, const float* __restrict__ k3,
                                      const float* __restrict__ k4, float dt, float* out, size_t n) {
    const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float third = static_cast<float>(1.0 / 3.0);
    float r;
    switch (mode) {
        case 0: r = __fadd_rn(y0[i], __fmul_rn(k1[i], dt)); break;
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

// qkv rows of timm's Attention (out-feature = which * D + head * dh + d, models/DiT.py:120 / SURVEY D6) re-ordered ONCE at upload
// into the head-major layout (head * 3 dhp + which * dhp + d) that the mma.sync attention kernels read (token grids other than 16 x 16,
// and head_dim 72).  dhp >= dh is the stored head width: DiT-XL's 72 channels are padded to 80 with zero rows, so q.k^T and P.V are
// unchanged and the padded output channels are exactly zero; the proj weight gets matching zero columns.
__global__ void dit_qkv_weight_repack_kernel(const float* __restrict__ w, __nv_bfloat16* __restrict__ out, int D, int dh, int dhp) {
    const int heads = D / dh;
    const size_t n = static_cast<size_t>(3) * heads * dhp * D;
    const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int r = static_cast<int>(i / D), k = static_cast<int>(i % D);
    const int h = r / (3 * dhp), which = (r % (3 * dhp)) / dhp, d = r % dhp;
    out[i] = d < dh ? __float2bfloat16(w[static_cast<size_t>(which * D + h * dh + d) * D + k]) : __float2bfloat16(0.f);
}
__global__ void dit_qkv_bias_repack_kernel(const float* __restrict__ b, float* __restrict__ out, int D, int dh, int dhp) {
    const int heads = D / dh;
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= 3 * heads * dhp) return;
    const int h = r / (3 * dhp), which = (r % (3 * dhp)) / dhp, d = r % dhp;
    out[r] = d < dh ? b[which * D + h * dh + d] : 0.f;
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
