"""The DiT's FP8 mode (lfm_set_fp8) against its bf16 path, in one run on an H100:
  1. the card's name and power limit;
  2. microseconds per launch of the qkv and fc1 GEMMs at M = 16384 (DiT-*/2 at batch 64): the bf16 kernel (lfm_dbg_gemm), the FP8
     kernel (lfm_dbg_gemm_fp8) and cuBLASLt's FP8 GEMM through torch._scaled_mm (row-wise scales where this torch takes them on
     sm_90, else per-tensor; the line says which; with and without fast accumulation), all with the bias epilogue and bf16 output
     (fc1's GELU only in ours);
  3. the per-kernel milliseconds per NFE of DiT-L/2 at batch 64 under torch.profiler, bf16 and FP8;
  4. Euler-50 sampling (step 0.02) of DiT-L/2 at batch 64, latents only, in images per second, alternating bf16 and FP8, twice each.
usage: fp8_profile.py [--out DIR]   (DIR/fp8_profile.json gets the numbers)"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import lfm_b200  # noqa: E402
from lfm_b200 import _lib  # noqa: E402
from lfm_b200.synthetic import synthetic_state_dict  # noqa: E402

PRESETS = {"S": (384, 384, 1536), "B": (768, 768, 3072), "L": (1024, 1024, 4096), "XL": (1152, 1280, 4608)}  # D, Dq, mlp hidden


def P(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def time_us(fn, iters=50, warmup=5):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / iters


def quantize_rows(v):
    amax = v.abs().amax(-1, keepdim=True)
    s = torch.where(amax > 0, amax / 448.0, torch.ones_like(amax))
    return (v / s).to(torch.float8_e4m3fn), s.squeeze(-1).contiguous()


def scaled_mm(qa, sa, qw, sw, bias, fast_accum=False):
    """cuBLASLt FP8: row-wise scales if accepted, else per-tensor.  Returns (callable, mode).  fast_accum=False (torch's default)
    has cuBLASLt promote the tensor cores' partial sums to fp32; True accumulates in the tensor cores, as our kernel does."""
    bt = qw.t()
    try:
        f = lambda: torch._scaled_mm(qa, bt, scale_a=sa[:, None], scale_b=sw[None, :], bias=bias, out_dtype=torch.bfloat16,  # noqa: E731
                                     use_fast_accum=fast_accum)
        f()
        torch.cuda.synchronize()
        return f, "row-wise"
    except (RuntimeError, ValueError):
        one = torch.ones((), device=qa.device)
        f = lambda: torch._scaled_mm(qa, bt, scale_a=one, scale_b=one, bias=bias, out_dtype=torch.bfloat16,  # noqa: E731
                                     use_fast_accum=fast_accum)
        f()
        torch.cuda.synchronize()
        return f, "per-tensor"


def gemm_rows(lib):
    M, out = 16384, []
    g = torch.Generator(device="cuda").manual_seed(0)
    for preset, (D, Dq, Hd) in PRESETS.items():
        for op, N, epi in (("qkv", 3 * Dq, 0), ("fc1", Hd, 1)):
            K = D
            a = torch.randn(M, K, device="cuda", generator=g)
            w = torch.randn(N, K, device="cuda", generator=g) * K ** -0.5
            bias = torch.randn(N, device="cuda", generator=g) * 0.1
            a16, w16 = a.bfloat16(), w.bfloat16()
            (qa, sa), (qw, sw) = quantize_rows(a), quantize_rows(w)
            o16 = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
            o8 = torch.empty_like(o16)
            us16 = time_us(lambda: lib.lfm_dbg_gemm(P(a16), P(w16), P(bias), P(o16), None, 0, 1, M, N, K, epi, 0, None))
            us8 = time_us(lambda: lib.lfm_dbg_gemm_fp8(P(qa), P(sa), P(qw), P(sw), P(bias), P(o8), M, N, K, epi, 0, None))
            f, mode = scaled_mm(qa, sa, qw, sw, bias.bfloat16())
            usc = time_us(f)
            f, _ = scaled_mm(qa, sa, qw, sw, bias.bfloat16(), fast_accum=True)
            usf = time_us(f)
            tflop = 2.0 * M * N * K / 1e12
            out.append(dict(preset=preset, op=op, M=M, N=N, K=K, us_bf16=round(us16, 1), us_fp8=round(us8, 1),
                            us_cublaslt_fp8=round(usc, 1), us_cublaslt_fp8_fast_accum=round(usf, 1), cublaslt_scales=mode,
                            tflops_bf16=round(tflop / us16 * 1e6, 1), tflops_fp8=round(tflop / us8 * 1e6, 1),
                            tflops_cublaslt_fp8=round(tflop / usc * 1e6, 1)))
            r = out[-1]
            print(f"{preset:>2} {op:<3} M {M} N {N} K {K}: bf16 {r['us_bf16']:7.1f} us ({r['tflops_bf16']} TFLOP/s)   "
                  f"fp8 {r['us_fp8']:7.1f} us ({r['tflops_fp8']})   cuBLASLt fp8 ({mode} scales, no GELU) {r['us_cublaslt_fp8']:7.1f} us "
                  f"({r['tflops_cublaslt_fp8']}), fast accumulation {usf:7.1f} us", flush=True)
            del a, w, a16, w16, qa, qw, o16, o8
    return out


def make_net(fp8, B):
    with torch.device("meta"):
        net = lfm_b200.DiT_models["DiT-L/2"](img_resolution=32, in_channels=4, label_dropout=0.0, num_classes=1, max_batch=B,
                                              fp8=fp8)
    sd = synthetic_state_dict(net, 1)
    net = net.to_empty(device="cpu")
    net.load_state_dict(sd, strict=True)
    return net.to("cuda").eval()


def kernel_table(net, x, iters=20):
    from torch.profiler import ProfilerActivity, profile
    t = torch.tensor(0.5, device="cuda")
    for _ in range(3):
        net(t, x)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            net(t, x)
        torch.cuda.synchronize()
    rows = {}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA or ev.name.startswith("Memcpy") or ev.name.startswith("Memset"):
            continue
        name = ev.name.removeprefix("void ").split("(")[0].removeprefix("lfm::")
        r = rows.setdefault(name, [0, 0.0])
        r[0] += 1
        r[1] += ev.device_time
    return {k: round(us / iters / 1e3, 3) for k, (n, us) in sorted(rows.items(), key=lambda kv: -kv[1][1])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fp8_profile.py measures on a CUDA device (H100); none is visible")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print("GPU:", gpu, flush=True)
    lib = _lib.load()
    res = {"gpu": gpu, "gemm_m16384": gemm_rows(lib)}

    B = 64
    x = torch.randn(B, 4, 32, 32, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    nets = {"bf16": make_net(False, B), "fp8": make_net(True, B)}
    res["dit_l2_b64_ms_per_nfe"] = {}
    for mode, net in nets.items():
        tab = kernel_table(net, x)
        res["dit_l2_b64_ms_per_nfe"][mode] = tab
        print(f"\nDiT-L/2 batch {B}, {mode}: kernel ms per NFE (torch.profiler), total {sum(tab.values()):.3f}")
        for k, v in tab.items():
            print(f"  {v:7.3f}  {k}")

    sargs = types.SimpleNamespace(method="euler", step_size=0.02, cfg_scale=1.0)
    for net in nets.values():                       # warm-up: step graphs captured
        lfm_b200.sample_from_model(net, x, {}, sargs)
    torch.cuda.synchronize()
    res["euler50_images_per_s"] = []
    for rep in range(2):
        for mode, net in nets.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            lfm_b200.sample_from_model(net, x, {}, sargs)
            e1.record()
            torch.cuda.synchronize()
            ips = B / (e0.elapsed_time(e1) / 1e3)
            res["euler50_images_per_s"].append({"mode": mode, "rep": rep, "images_per_s": round(ips, 2)})
            print(f"Euler-50 DiT-L/2 batch {B} {mode} (run {rep + 1}): {ips:.2f} images/s", flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "fp8_profile.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
