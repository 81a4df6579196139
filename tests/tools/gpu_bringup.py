"""GPU bring-up diagnostics (run on an H100):  python tests/tools/gpu_bringup.py <group>
Groups: gemm, attn, forward, sampler, perf.  Prints error statistics; used to localise kernel bugs."""
import ctypes as C
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from lfm_b200 import _lib  # noqa: E402

lib = _lib.load()
dev = torch.device("cuda:0")


def P(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def stats(name, got, ref):
    got, ref = got.double(), ref.double()
    err = (got - ref).abs()
    rel = float((got - ref).norm() / ref.norm().clamp_min(1e-30))
    print(f"  {name}: rel_l2={rel:.3e} max_abs={float(err.max()):.3e} ref_absmax={float(ref.abs().max()):.3e} "
          f"nan={int(torch.isnan(got).sum())}", flush=True)
    return rel


def gemm_case(M, N, K, epi, bn, T=256, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    a = (torch.randn(M, K, generator=g) * 0.5).to(dev).bfloat16()
    w = (torch.randn(N, K, generator=g) * 0.05).to(dev).bfloat16()
    bias = torch.randn(N, generator=g).to(dev)
    acc = a.float() @ w.float().t() + bias
    nb = (M + T - 1) // T
    gate = torch.randn(nb, 3 * N, generator=g).to(dev)
    if epi == 0:
        out = torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
        ref = acc
    elif epi == 1:
        out = torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
        ref = torch.nn.functional.gelu(acc, approximate="tanh")
    elif epi == 2:
        x0 = torch.randn(M, N, generator=g).to(dev)
        out = x0.clone()
        rows = torch.arange(M, device=dev) // T
        ref = x0 + gate[rows, N:2 * N] * acc
    else:
        out = torch.zeros(M, N, device=dev, dtype=torch.float32)
        ref = acc
    rc = lib.lfm_dbg_gemm(P(a), P(w), P(bias), P(out), C.c_void_p(gate.data_ptr() + N * 4), 3 * N, T, M, N, K, epi, bn, None)
    torch.cuda.synchronize()
    if rc:
        print("  rc", rc, _lib.last_error())
        return 1.0
    return stats(f"gemm M={M} N={N} K={K} epi={epi} bn={bn}", out.float(), ref)


def group_gemm():
    for (M, N, K, epi, bn) in [(128, 128, 64, 3, 128), (128, 256, 64, 3, 256), (256, 256, 128, 3, 256),
                               (256, 512, 1024, 0, 256), (512, 1024, 1024, 1, 256), (512, 1024, 4096, 2, 256),
                               (512, 1024, 4096, 2, 128), (64, 2048, 1024, 3, 256), (4, 1024, 256, 3, 256),
                               (256, 1152, 384, 0, 256), (256, 1152, 384, 0, 128), (16384, 3072, 1024, 0, 256),
                               (16384, 1024, 1024, 2, 128),
                               (256, 256, 64, 3, 0), (256, 512, 1024, 0, 0), (512, 1024, 1024, 1, 0),
                               (512, 1024, 4096, 2, 0), (64, 2048, 1024, 3, 0), (768, 1152, 384, 0, 0),
                               (16384, 3072, 1024, 0, 0), (16384, 1024, 4096, 2, 0), (16384, 4096, 1024, 1, 0)]:
        gemm_case(M, N, K, epi, bn)


def group_gemm4():
    for (M, N, K, epi) in [(256, 512, 64, 3), (256, 512, 1024, 0), (512, 1024, 4096, 2), (768, 768, 384, 1), (16384, 3072, 1024, 0),
                           (16384, 1024, 4096, 2), (16384, 4096, 1024, 1), (16384, 1024, 1024, 2)]:
        gemm_case(M, N, K, epi, 0)
    for (N, K, epi) in ((3072, 1024, 0), (1024, 1024, 2), (4096, 1024, 1), (1024, 4096, 2)):
        time_gemm(16384, N, K, epi, 0)


def attn_ref(qkv, B, H):
    D = H * 64
    q, k, v = qkv.float().reshape(B, 256, 3, H, 64).permute(2, 0, 3, 1, 4)
    s = q @ k.transpose(-1, -2)
    p = torch.softmax(s * 0.125, dim=-1)
    o = (p @ v).transpose(1, 2).reshape(B * 256, D)
    return s, o


def head_major(qkv, B, H):
    """The same q, k, v with the rows of each token in head-major order (head * 192 + {q,k,v} * 64 + c)."""
    return qkv.reshape(B * 256, 3, H, 64).transpose(1, 2).reshape(B * 256, 3 * H * 64).contiguous()


def group_attn():
    B, H = 2, 4
    D = H * 64
    g = torch.Generator().manual_seed(3)
    qkv = (torch.randn(B * 256, 3 * D, generator=g)).to(dev).bfloat16()
    s_ref, o_ref = attn_ref(qkv, B, H)
    for layout in (_lib.QKV_TIMM, _lib.QKV_HEAD_MAJOR):   # the TMA + wgmma route, the flash route
        src = qkv if layout == _lib.QKV_TIMM else head_major(qkv, B, H)
        out = torch.zeros(B * 256, D, device=dev, dtype=torch.bfloat16)
        rc = lib.lfm_dbg_attention(P(src), P(out), B, 256, H, 64, 64, layout, None)
        torch.cuda.synchronize()
        print(f" attention layout {layout} rc={rc} {_lib.last_error() if rc else ''}")
        stats("O", out.float(), o_ref)
        # per-q-tile / per-column-block diagnostics
        e = (out.float() - o_ref).abs().reshape(B, 2, 128, H, 64)
        print("   err by (qtile):", e.amax(dim=(0, 2, 3, 4)).tolist(), " by head:", e.amax(dim=(0, 1, 2, 4)).tolist())
    B, H = 64, 16
    D = H * 64
    qkv = (torch.randn(B * 256, 3 * D, generator=g)).to(dev).bfloat16()
    _, o_ref = attn_ref(qkv, B, H)
    for layout in (_lib.QKV_TIMM, _lib.QKV_HEAD_MAJOR):
        src = qkv if layout == _lib.QKV_TIMM else head_major(qkv, B, H)
        out = torch.zeros(B * 256, D, device=dev, dtype=torch.bfloat16)
        lib.lfm_dbg_attention(P(src), P(out), B, 256, H, 64, 64, layout, None)
        torch.cuda.synchronize()
        stats(f"O full B=64 H=16 layout {layout}", out.float(), o_ref)
        t0 = torch.cuda.Event(enable_timing=True); t1 = torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(10):
            lib.lfm_dbg_attention(P(src), P(out), B, 256, H, 64, 64, layout, None)
        t1.record(); torch.cuda.synchronize()
        ms = t0.elapsed_time(t1) / 10
        print(f"   attention B=64 H=16 layout {layout}: {ms*1e3:.1f} us  ({4*256*256*64*B*H/ms/1e9:.1f} TFLOP/s)")


def group_forward():
    import lfm_b200
    from oracle import dit as odit
    from tests._util import T, cfg_from_golden, load_golden, rel_l2
    for name in ("mini_uncond", "mini_cond", "mini_d384"):
        g = load_golden(name)
        cfg = cfg_from_golden(g)
        sd = odit.synthetic_state_dict(cfg, int(g["weight_seed"]))
        net = lfm_b200.DiT(img_resolution=32, patch_size=2, in_channels=4, hidden_size=cfg.hidden_size, depth=cfg.depth,
                           num_heads=cfg.num_heads, label_dropout=cfg.label_dropout, num_classes=cfg.num_classes)
        net.load_state_dict(sd, strict=True)
        net = net.to(dev)
        x = T(g["x"]).to(dev)
        v = net(T(g["t_scalar"]).to(dev), x)
        torch.cuda.synchronize()
        stats(f"{name} forward scalar-t y=None", v.cpu(), T(g["v_scalar_ynone"]))
        # token stream vs oracle for localisation
        tok = torch.empty(2 * 256 * cfg.hidden_size, device=dev)
        lib.lfm_dbg_tokens(net._ctx, P(tok), 2)
        tok_ref = odit.dit_forward(sd, cfg, T(g["t_scalar"]), T(g["x"]), None, return_tokens=True)
        stats(f"{name} token stream", tok.cpu().reshape(tok_ref.shape), tok_ref)
        v = net(T(g["t_vec"]).to(dev), x, T(g["y"]).to(dev))
        stats(f"{name} forward vec-t y", v.cpu(), T(g["v_vec_y"]))
        if cfg.num_classes > 1:
            v = net.forward_with_cfg(torch.full((4,), 0.4, device=dev), torch.cat([x, x]), T(g["y_cfg"]).to(dev), 1.5)
            stats(f"{name} forward_with_cfg", v.cpu(), T(g["v_cfg_1p5"]))


def group_sampler():
    import lfm_b200
    from oracle import dit as odit
    from tests._util import T, cfg_from_golden, load_golden
    for name in ("mini_uncond", "mini_cond"):
        g = load_golden(name)
        cfg = cfg_from_golden(g)
        sd = odit.synthetic_state_dict(cfg, int(g["weight_seed"]))
        net = lfm_b200.DiT(img_resolution=32, patch_size=2, in_channels=4, hidden_size=cfg.hidden_size, depth=cfg.depth,
                           num_heads=cfg.num_heads, label_dropout=cfg.label_dropout, num_classes=cfg.num_classes)
        net.load_state_dict(sd, strict=True)
        net = net.to(dev)
        x = T(g["x"]).to(dev)
        if cfg.num_classes > 1:
            xs, mk = torch.cat([x, x]), dict(y=T(g["y_cfg"]).to(dev), cfg_scale=1.5)
        else:
            xs, mk = x, {}
        for smp, key, steps in (("euler", "euler6", 6), ("heun", "heun5", 5)):
            out = lfm_b200.karras_sample(net, xs, steps, clip_denoised=False, model_kwargs=mk, sigma_min=1e-5, sigma_max=1.0,
                                         sampler=smp)
            torch.cuda.synchronize()
            stats(f"{name} karras {smp} steps={steps} nfe={net.last_stats}", out.cpu(), T(g[key]))
        if name == "mini_uncond":
            out = lfm_b200.karras_sample(net, xs, 43, clip_denoised=False, model_kwargs=mk, sigma_min=1e-5, sigma_max=1.0,
                                         sampler="heun")
            stats(f"{name} heun43 nfe={net.last_stats}", out.cpu(), T(g["heun43"]))
            import types
            args = types.SimpleNamespace(method="dopri5", atol=1e-5, rtol=1e-5, cfg_scale=1.0, compute_nfe=True)
            traj, nfe = lfm_b200.sample_from_model(net, xs, {}, args)
            from oracle import solvers as osol
            from tests._util import oracle_model
            ref, st = osol.tdq_dopri5(oracle_model(sd, cfg), T(g["x"]))
            stats(f"dopri5 nfe={net.last_stats} oracle nfe={st.nfe}/{st.accepted}/{st.rejected}", traj[-1].cpu(), ref)
            args = types.SimpleNamespace(method="euler", step_size=0.1, perturb=False, cfg_scale=1.0, compute_nfe=False)
            traj = lfm_b200.sample_from_model(net, xs, {}, args)
            ref, n = osol.tdq_euler(oracle_model(sd, cfg), T(g["x"]), 0.1)
            stats(f"tdq euler h=0.1 nfe={net.last_stats}", traj[-1].cpu(), ref)


def group_unet():
    import types
    import lfm_b200
    from oracle import unet as ounet
    from oracle import solvers as osol
    from tests._util import T, load_golden
    from tests.test_oracle_unet import unet_cfg_from_golden
    for name in ("unet_mini", "unet_mini_cond", "unet_celeb256"):
        g = load_golden(name)
        cfg = unet_cfg_from_golden(g) if name != "unet_celeb256" else ounet.UNetConfig(image_size=32, channel_mult=(1, 2, 2, 2))
        sd = ounet.synthetic_state_dict(cfg, int(g["weight_seed"]))
        net = lfm_b200.UNetModel(image_size=cfg.image_size, in_channels=4, model_channels=cfg.model_channels, out_channels=4,
                                 num_res_blocks=cfg.num_res_blocks, attention_resolutions=cfg.attention_resolutions,
                                 channel_mult=cfg.channel_mult, num_classes=cfg.num_classes, num_heads=cfg.num_heads,
                                 num_head_channels=cfg.num_head_channels, use_scale_shift_norm=True)
        net.load_state_dict(sd, strict=True)
        net = net.to(dev)
        x = T(g["x"]).to(dev)
        y = T(g["y"]).to(dev) if "y" in g else None
        v = net(T(g["t_vec"]).to(dev), x, y)
        torch.cuda.synchronize()
        stats(f"{name} forward", v.cpu(), T(g["v"]))
        e = (v.cpu() - T(g["v"])).abs()
        print("   err by sample:", e.amax(dim=(1, 2, 3)).tolist(), " by channel:", e.amax(dim=(0, 2, 3)).tolist())
        if name == "unet_mini":
            args = types.SimpleNamespace(method="dopri5", atol=1e-3, rtol=1e-3, cfg_scale=1.0, compute_nfe=True)
            traj, nfe = lfm_b200.sample_from_model(net, x, {}, args)
            ref, st = osol.tdq_dopri5(lambda tt, xx: ounet.unet_forward(sd, cfg, tt, xx), T(g["x"]), rtol=1e-3, atol=1e-3)
            stats(f"unet dopri5 nfe={net.last_stats} oracle={st.nfe}/{st.accepted}/{st.rejected}", traj[-1].cpu(), ref)
            out = lfm_b200.karras_sample(net, x, 4, clip_denoised=False, model_kwargs={}, sigma_min=1e-5, sigma_max=1.0, sampler="heun")
            ref = osol.karras_sample(lambda tt, xx: ounet.unet_forward(sd, cfg, tt, xx), T(g["x"]), 4, "heun")
            stats(f"unet heun4 nfe={net.last_stats}", out.cpu(), ref)
    # celeb512 preset timing, B=8
    cfg = ounet.UNetConfig()
    with torch.device("meta"):
        net = lfm_b200.UNetModel(image_size=64, in_channels=4, model_channels=256, out_channels=4, num_res_blocks=2,
                                 attention_resolutions=(16, 8), channel_mult=(1, 2, 2, 2, 4), num_heads=4, use_scale_shift_norm=True)
    from lfm_b200.synthetic import synthetic_unet_state_dict
    sd = synthetic_unet_state_dict(net, 1)
    net = net.to_empty(device="cpu"); net.load_state_dict(sd, strict=True); net = net.to(dev)
    for B in (8, 32):
        x = torch.randn(B, 4, 64, 64, device=dev)
        t = torch.tensor(0.5, device=dev)
        for _ in range(2):
            v = net(t, x)
        torch.cuda.synchronize()
        t0 = torch.cuda.Event(enable_timing=True); t1 = torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(5):
            v = net(t, x)
        t1.record(); torch.cuda.synchronize()
        ms = t0.elapsed_time(t1) / 5
        fl = ounet.unet_flops_per_sample(cfg) * B
        print(f"  celeb512 UNet forward B={B}: {ms:.2f} ms  {fl/ms/1e9:.1f} TFLOP/s  finite={bool(torch.isfinite(v).all())} absmean={float(v.abs().mean()):.4f}")
        if B == 8:
            ref = ounet.unet_forward(sd, cfg, torch.tensor(0.5), x[:1].cpu())
            stats("celeb512 B=8 sample 0 vs oracle", v[:1].cpu(), ref)


def time_gemm(M, N, K, epi, bn, iters=20):
    a = torch.randn(M, K, device=dev).bfloat16()
    w = (torch.randn(N, K, device=dev) * 0.05).bfloat16()
    bias = torch.randn(N, device=dev)
    gate = torch.randn((M + 255) // 256, N, device=dev)
    out = torch.zeros(M, N, device=dev, dtype=torch.float32 if epi >= 2 else torch.bfloat16)
    for _ in range(3):
        lib.lfm_dbg_gemm(P(a), P(w), P(bias), P(out), P(gate), N, 256, M, N, K, epi, bn, None)
    t0 = torch.cuda.Event(enable_timing=True); t1 = torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        lib.lfm_dbg_gemm(P(a), P(w), P(bias), P(out), P(gate), N, 256, M, N, K, epi, bn, None)
    t1.record(); torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / iters
    print(f"  gemm M={M} N={N} K={K} epi={epi} bn={bn}: {ms*1e3:8.1f} us  {2*M*N*K/ms/1e9:8.1f} TFLOP/s", flush=True)


def group_perf16k():
    for (N, K, epi) in ((3072, 1024, 0), (1024, 1024, 2), (4096, 1024, 1), (1024, 4096, 2)):
        time_gemm(16384, N, K, epi, 0)


def group_perf():
    for M in (16384, 32768, 4096):
        for (N, K, epi) in ((3072, 1024, 0), (1024, 1024, 2), (4096, 1024, 1), (1024, 4096, 2)):
            time_gemm(M, N, K, epi, 0)
    # cuBLAS reference for the same shapes
    for (M, N, K) in ((16384, 3072, 1024), (16384, 1024, 1024), (16384, 4096, 1024), (16384, 1024, 4096)):
        a = torch.randn(M, K, device=dev).bfloat16(); w = torch.randn(N, K, device=dev).bfloat16()
        for _ in range(3):
            a @ w.t()
        t0 = torch.cuda.Event(enable_timing=True); t1 = torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(20):
            a @ w.t()
        t1.record(); torch.cuda.synchronize()
        ms = t0.elapsed_time(t1) / 20
        print(f"  cuBLAS M={M} N={N} K={K}: {ms*1e3:8.1f} us {2*M*N*K/ms/1e9:8.1f} TFLOP/s")


if __name__ == "__main__":
    grp = sys.argv[1]
    print(f"=== {grp} ===", flush=True)
    t = time.time()
    {"gemm": group_gemm, "attn": group_attn, "forward": group_forward, "sampler": group_sampler, "perf": group_perf, "unet": group_unet, "gemm4": group_gemm4, "perf16k": group_perf16k}[grp]()
    print(f"=== {grp} done in {time.time()-t:.1f}s ===", flush=True)
