// lfm_b200 - kernels of the native VAE decode and encode (Stable-Diffusion AutoencoderKL; reference call sites
// test_flow_latent.py:193 `first_stage_model.decode(fake_sample / args.scale_factor).sample` and
// downstream_tasks/test_flow_latent_inpainting.py:147 `first_stage_model.encode(masked_image).latent_dist`) that are not the
// shared implicit-GEMM convolution / GroupNorm kernels of unet.cuh, and the device side of the generation loop's
// post-processing (test_flow_latent_ddp.py:131-135).
#pragma once
#include "common.cuh"

namespace lfm {

// post_quant_conv: 1x1 convolution 4 -> 4 on the NCHW fp32 latents (AutoencoderKL.decode, before the decoder).
__global__ void vae_post_quant_kernel(const float* __restrict__ z, const float* __restrict__ W /*[4][4]*/, const float* __restrict__ bias,
                                      float* __restrict__ out, int B, int HW) {
    pdl_wait();
    pdl_trigger();
    const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= static_cast<size_t>(B) * HW) return;
    const size_t b = i / HW, p = i % HW;
    const float* zp = z + b * 4 * HW + p;
    const float v0 = zp[0], v1 = zp[HW], v2 = zp[2 * static_cast<size_t>(HW)], v3 = zp[3 * static_cast<size_t>(HW)];
    float* op = out + b * 4 * HW + p;
#pragma unroll
    for (int o = 0; o < 4; ++o)
        op[static_cast<size_t>(o) * HW] = fmaf(W[o * 4 + 3], v3, fmaf(W[o * 4 + 2], v2, fmaf(W[o * 4 + 1], v1, fmaf(W[o * 4], v0, bias[o]))));
}

// AutoencoderKL.encode's tail: quant_conv (1x1, 8 -> 8) on the encoder's conv_out, NHWC fp32 [B*HW, 8], then the moments of
// DiagonalGaussianDistribution: mean = channels 0..3 and logvar = clamp(channels 4..7, -30, 20), both NCHW fp32 [B, 4, HW].
// Each output is the bias plus the channels in order, one fma each.
__global__ void vae_quant_kernel(const float* __restrict__ in /*[B*HW, 8]*/, const float* __restrict__ W /*[8][8]*/,
                                 const float* __restrict__ bias, float* __restrict__ mean, float* __restrict__ logvar, int B, int HW) {
    pdl_wait();
    pdl_trigger();
    const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= static_cast<size_t>(B) * HW) return;
    const float4 lo = *reinterpret_cast<const float4*>(in + i * 8), hi = *reinterpret_cast<const float4*>(in + i * 8 + 4);
    const float v[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
    const size_t b = i / HW, p = i % HW;
#pragma unroll
    for (int o = 0; o < 8; ++o) {
        float acc = bias[o];
#pragma unroll
        for (int c = 0; c < 8; ++c) acc = fmaf(W[o * 8 + c], v[c], acc);
        if (o < 4)
            mean[(b * 4 + o) * HW + p] = acc;
        else
            logvar[(b * 4 + o - 4) * HW + p] = fminf(fmaxf(acc, -30.0f), 20.0f);
    }
}

// Row softmax of the mid-block attention: P = softmax(S * scale) over the last dimension, S fp32 [R, 128 NV] (the
// output of the batched Q K^T GEMM) -> P bf16 (A operand of the P V GEMM).  One warp per row, the row lives in
// registers (NV float4 per lane), exp2 with the scale folded into the exponent.
template <int NV>
__global__ void __launch_bounds__(256)
softmax_rows_kernel(const float* __restrict__ S, __nv_bfloat16* __restrict__ P, int R, float scale_log2e) {
    pdl_wait();
    pdl_trigger();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    constexpr int T = NV * 128;
    for (int r = blockIdx.x * 8 + warp; r < R; r += gridDim.x * 8) {
        const float4* sp = reinterpret_cast<const float4*>(S + static_cast<size_t>(r) * T);
        float4 v[NV];
#pragma unroll
        for (int j = 0; j < NV; ++j) v[j] = sp[j * 32 + lane];
        float mx = -INFINITY;
#pragma unroll
        for (int j = 0; j < NV; ++j) mx = fmaxf(mx, fmaxf(fmaxf(v[j].x, v[j].y), fmaxf(v[j].z, v[j].w)));
        mx = warp_max(mx) * scale_log2e;
        float sum = 0.f;
#pragma unroll
        for (int j = 0; j < NV; ++j) {
            v[j].x = exp2f(fmaf(v[j].x, scale_log2e, -mx));
            v[j].y = exp2f(fmaf(v[j].y, scale_log2e, -mx));
            v[j].z = exp2f(fmaf(v[j].z, scale_log2e, -mx));
            v[j].w = exp2f(fmaf(v[j].w, scale_log2e, -mx));
            sum += (v[j].x + v[j].y) + (v[j].z + v[j].w);
        }
        const float inv = 1.f / warp_sum(sum);
        uint2* pp = reinterpret_cast<uint2*>(P + static_cast<size_t>(r) * T);
#pragma unroll
        for (int j = 0; j < NV; ++j)
            pp[j * 32 + lane] = make_uint2(pack_bf16x2(v[j].x * inv, v[j].y * inv), pack_bf16x2(v[j].z * inv, v[j].w * inv));
    }
}

// conv_out writes NHWC with 4 columns (3 image channels + one zero column of the padded GEMM); this produces what the
// callers consume: `sample` fp32 NCHW [B, 3, H, W] (AutoencoderKL.decode(...).sample) and / or the post-processed image
// uint8 NHWC [B, H, W, 3] = (clamp((x + 1) / 2, 0, 1) * 255).permute(0, 2, 3, 1).to(uint8)  (truncation, as torch).
__global__ void vae_image_out_kernel(const float* __restrict__ in /*[B*HW, 4]*/, float* __restrict__ out_f32, uint8_t* __restrict__ out_u8,
                                     int B, int HW) {
    pdl_wait();
    pdl_trigger();
    const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= static_cast<size_t>(B) * HW) return;
    const float4 v = *reinterpret_cast<const float4*>(in + i * 4);
    const size_t b = i / HW, p = i % HW;
    if (out_f32 != nullptr) {
        float* o = out_f32 + b * 3 * HW + p;
        o[0] = v.x;
        o[HW] = v.y;
        o[2 * static_cast<size_t>(HW)] = v.z;
    }
    if (out_u8 != nullptr) {
        const float c[3] = {v.x, v.y, v.z};
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const float t = __fmul_rn(fminf(fmaxf(__fmul_rn(__fadd_rn(c[k], 1.0f), 0.5f), 0.0f), 1.0f), 255.0f);
            out_u8[i * 3 + k] = static_cast<uint8_t>(static_cast<int>(t));  // t in [0, 255]: truncation toward zero
        }
    }
}

}  // namespace lfm
