#!/usr/bin/env python
"""bench.py - headline benchmark of the H100-native LFM sampling path.

    python bench.py --gpus N --steps K --warmup W            # ours (one process per GPU under torchrun for N > 1)
    python bench.py --impl reference --gpus N --steps K --warmup W   # the reference algorithm on the host CPU
    python bench.py ... --dump-outputs DIR    # also write the last timed step's sampled latents to DIR/latents.npy

Workload (BASELINE.json configs[1]): DiT-L/2, 32x32x4 latents, Euler-50 (torchdiffeq-style uniform grid,
step_size 0.02 => 50 NFE), batch 64 per GPU, synthetic non-degenerate weights (lfm_b200.synthetic
seed 1 - the reference's own init is all-zero at the output) and Gaussian latents.  One "step" = one full
sampling pass over one batch of 64 latents per GPU.  Metric: images/s (whole job, weak scaling).

After the headline region the same process also measures, and reports under extra keys of the SAME line:
`other_configs` (BASELINE.json configs 3, 4, 5 at this GPU count: DiT-B/2 CFG Heun-25, ADM UNet dopri5 1e-5 at N=1,
DiT-L/2 batch-128 Euler sweep in weak and strong scaling; at N=1 also DiT-XL/2 and DiT-L/2 on 64x64 latents), `gemm_vs_cublas` (the four DiT-L GEMM shapes, our kernel
vs torch.matmul on the same box), `gpu_eager_baseline` (the reference network in eager PyTorch on this GPU: bf16
autocast + SDPA + TF32) and `decode` (images/s including the native VAE decode).  `--no-extras` skips them.

Prints ONE JSON line (rank 0).  See DESIGN.md "Measurement" for every field.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import threading
import time
import types

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

DEFAULT_GEMM_BN = 256   # lfm_dbg_gemm tile width of the GEMM kernel (128 x 256 tiles, the network's choice for these shapes)
MODEL = "DiT-L/2"
BATCH = 64
NFE = 50
STEP_SIZE = 1.0 / NFE
WEIGHT_SEED = 1


def load_peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        with open(p) as f:
            d = json.load(f)
        return dict(burst=float(d["bf16_tflops"]), sustained=float(d.get("bf16_tflops_sustained", d["bf16_tflops"])),
                    hbm=float(d["hbm_gbs"]), source="measured (MEASURED_PEAKS.json)")
    # NVIDIA H100 SXM data sheet (700 W board): dense BF16 989 TFLOP/s, HBM3 3.35 TB/s - a ceiling, not a measured rate
    return dict(burst=989.0, sustained=989.0, hbm=3350.0, source="fallback (H100 SXM data sheet, dense BF16)")


class ClockSampler:
    """nvidia-smi clocks / throttle reasons sampled every 200 ms while the timed region runs."""
    Q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, index):
        self.index, self.rows, self.proc, self.thr = index, [], None, None

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.index), f"--query-gpu={self.Q}",
                                          "--format=csv,noheader,nounits", "-lms", "200"], stdout=subprocess.PIPE,
                                         stderr=subprocess.DEVNULL, text=True)
        except OSError:
            self.proc = None
            return
        self.thr = threading.Thread(target=self._read, daemon=True)
        self.thr.start()

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([c.strip() for c in line.split(",")])

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()  # the exact child we started
        try:
            self.proc.wait(timeout=5)
        except subprocess.TimeoutExpired:
            self.proc.kill()
        sm, smax, reasons, power = [], None, set(), []
        for r in self.rows:
            try:
                sm.append(float(r[0]))
                smax = float(r[1])
                power.append(float(r[2]))
            except (ValueError, IndexError):
                continue
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), r[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        busy = [c for c in sm if smax and c > 0.3 * smax] or sm
        return {"sm_mhz": statistics.median(busy) if busy else None, "sm_max_mhz": smax, "reasons": sorted(reasons),
                "power_w_max": max(power) if power else None, "samples": len(sm)}


def build_model(device, model=MODEL, num_classes=1, label_dropout=0.0, max_batch=BATCH, latent_side=32):
    import lfm_b200
    from lfm_b200.synthetic import synthetic_state_dict
    with torch.device("meta"):
        net = lfm_b200.DiT_models[model](img_resolution=latent_side, in_channels=4, label_dropout=label_dropout, num_classes=num_classes)
    sd = synthetic_state_dict(net, WEIGHT_SEED)
    net = net.to_empty(device="cpu")
    net.load_state_dict(sd, strict=True)
    net = net.to(device)
    net.max_batch_hint = max_batch
    return net


def build_unet_celeb512(device, max_batch):
    import lfm_b200
    from lfm_b200.synthetic import synthetic_unet_state_dict
    with torch.device("meta"):
        net = lfm_b200.UNetModel(image_size=64, in_channels=4, model_channels=256, out_channels=4, num_res_blocks=2,
                                 attention_resolutions=(16, 8), channel_mult=(1, 2, 2, 2, 4), num_heads=4,
                                 use_scale_shift_norm=True, max_batch=max_batch)
    sd = synthetic_unet_state_dict(net, WEIGHT_SEED)
    net = net.to_empty(device="cpu")
    net.load_state_dict(sd, strict=True)
    return net.to(device)


def time_dominant_kernel(device, peaks, iters=20):
    """Roofline of the dominant kernel: the wgmma GEMM (gemm_bf16_wgmma), on its largest instance in the network
    (mlp.fc1 + bias + GELU: M = 64*256, N = 4096, K = 1024), timed with CUDA events on the launching stream.
    Operands + output = 176 MB > the 50 MB L2."""
    from lfm_b200 import _lib
    lib = _lib.load()
    M, N, K = BATCH * 256, 4096, 1024
    a = torch.randn(M, K, device=device).bfloat16()
    w = (torch.randn(N, K, device=device) * 0.03).bfloat16()
    bias = torch.randn(N, device=device)
    out = torch.empty(M, N, device=device, dtype=torch.bfloat16)
    s = C.c_void_p(torch.cuda.current_stream(device).cuda_stream)

    def run():
        rc = lib.lfm_dbg_gemm(a.data_ptr(), w.data_ptr(), bias.data_ptr(), out.data_ptr(), None, 0, 256, M, N, K, 1, DEFAULT_GEMM_BN, s)
        assert rc == 0, _lib.last_error()
    for _ in range(3):
        run()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize(device)
    e0.record()
    for _ in range(iters):
        run()
    e1.record()
    torch.cuda.synchronize(device)
    ms = e0.elapsed_time(e1) / iters
    achieved = 2.0 * M * N * K / (ms * 1e-3) / 1e12
    return {"bound": "tensor", "kernel": "gemm_bf16_wgmma<256, EPI_BIAS_GELU_BF16> (128x256 tile) M=16384 N=4096 K=1024",
            "achieved": round(achieved, 1), "peak": peaks["burst"], "unit": "TFLOP/s", "frac": round(achieved / peaks["burst"], 4),
            "us_per_launch": round(ms * 1e3, 2), "peak_source": peaks["source"] + ", burst (kernel timed alone)"}


def usable_threads():
    """Host threads the CPU legs should use.  os.cpu_count() reports the machine (128 on the GPU box) while the
    container may be entitled to far fewer cores; oversubscribing MKL there is ~50x slower.  Calibrate: time a
    1024^3 fp32 matmul at a few thread counts and keep the fastest."""
    try:
        avail = len(os.sched_getaffinity(0))
    except AttributeError:
        avail = os.cpu_count() or 1
    a = torch.randn(1024, 1024)
    best, best_t = 1, float("inf")
    cand = sorted({c for c in (4, 8, 16, 32, 64, 128, avail) if c <= avail})
    for c in cand:
        torch.set_num_threads(c)
        a @ a
        t0 = time.perf_counter()
        for _ in range(3):
            a @ a
        dt = time.perf_counter() - t0
        if dt < best_t * 0.9:
            best, best_t = c, dt
    torch.set_num_threads(best)
    return best


def cpu_baseline(threads, seconds_hint=20):
    """The oracle (CPU port of the reference algorithm, fp32) on the host cores, bounded sample."""
    from oracle import dit as odit
    from oracle import solvers as osol
    torch.set_num_threads(threads)
    cfg = odit.make_config(MODEL, num_classes=1, label_dropout=0.0)
    sd = odit.synthetic_state_dict(cfg, WEIGHT_SEED)
    B = 4   # the CPU is most efficient at small batches (measured: batch 16 halves its NFE*img/s)
    x = torch.randn(B, 4, 32, 32, generator=torch.Generator().manual_seed(0))
    f = lambda t, xx: odit.dit_forward(sd, cfg, t, xx)  # noqa: E731
    osol.tdq_euler(f, x, 1.0)  # warm-up: 1 NFE
    t0 = time.time()
    _, nfe = osol.tdq_euler(f, x, 0.04)  # bounded sample of the workload: 25 of the 50 Euler steps, batch 4 (~10-20 s)
    dt = time.time() - t0
    return B * nfe / dt / NFE, dt, f"DiT-L/2 fp32 oracle, batch {B}, {nfe} Euler NFE in {dt:.2f}s, scaled to Euler-{NFE} images/s"


def workload_config(world):
    """The `config` object of the GPU arm."""
    return {"workload": f"{MODEL} 32x32x4 latents, Euler-{NFE} (step_size {STEP_SIZE}), batch {BATCH}/GPU, "
                        f"synthetic non-degenerate init (seed {WEIGHT_SEED}), {'dp' + str(world)}",
            "l2": "inputs larger than L2: 0.9 GB of weights + 0.7 GB of activations stream per NFE (L2 = 50 MB)",
            "global_batch": BATCH * world, "nfe_per_image": NFE}


# The reference arm's "step" is a bounded sample of one pass: REF_NFE_PER_STEP of its 50 Euler NFE on REF_BATCH of its 64
# latents (the driver runs --steps 20 --warmup 5; a full-batch NFE takes 5-15 s on the box's host cores).  The CPU's
# NFE x images / s does not grow with the batch (measured: batch 16 is no faster per image than batch 4).
REF_NFE_PER_STEP = 1
REF_BATCH = 16


def run_reference(args):
    """--impl reference: the reference algorithm (oracle port; the reference is pure Python + absent dependencies and
    cannot travel to the GPU box) on the host CPU with all the threads it can use; rank 0 only.  Same workload as the
    GPU arm - DiT-L/2, Euler-50, fp32 - but one step is a BOUNDED SAMPLE of it: REF_NFE_PER_STEP of the 50 Euler
    network evaluations of a pass on REF_BATCH of the 64 latents (every NFE costs the same, so
    images/s = REF_BATCH x NFE_run / (50 x step seconds)); the config object says so."""
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    threads = usable_threads()
    from oracle import dit as odit
    from oracle import solvers as osol
    cfg = odit.make_config(MODEL, num_classes=1, label_dropout=0.0)
    sd = odit.synthetic_state_dict(cfg, WEIGHT_SEED)
    B, nfe_s = REF_BATCH, REF_NFE_PER_STEP
    x = torch.randn(B, 4, 32, 32, generator=torch.Generator().manual_seed(0))
    f = lambda t, xx: odit.dit_forward(sd, cfg, t, xx)  # noqa: E731
    for _ in range(max(1, min(args.warmup, 2))):
        osol.tdq_euler(f, x, 1.0 / nfe_s)
    t0 = time.time()
    for _ in range(args.steps):
        osol.tdq_euler(f, x, 1.0 / nfe_s)
    dt = (time.time() - t0) / args.steps
    value = B * nfe_s / dt / NFE
    sample = (f"each step = {nfe_s} of the {NFE} Euler NFE of one pass on {B} of the {BATCH} latents: DiT-L/2 fp32 oracle port, on "
              f"{threads} host threads ({dt:.2f} s per step); images/s = {B} x {nfe_s} / (step time x {NFE})")
    conf = workload_config(int(os.environ.get("WORLD_SIZE", "1")))
    conf["workload"] = (f"{MODEL} 32x32x4 latents, Euler-{NFE} metric measured on a bounded sample: batch {B}, {nfe_s} Euler NFE per "
                        f"step, fp32, host CPU ({threads} threads), rank 0 only; scaled to Euler-{NFE} images/s")
    conf["global_batch"] = B
    conf["reference_step"] = sample
    line = {"impl": "reference", "metric": "images/sec DiT-L/2 32x32 latents Euler-50", "value": value, "unit": "images/s",
            "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup, "ms_per_step": dt * 1e3,
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": conf,
            "cpu_baseline": {"value": value, "unit": "images/s", "cores": threads, "kind": "port", "sample": sample},
            "e2e": {"value": value, "unit": "images/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
            "gpu_launches": 0}
    print(json.dumps(line), flush=True)


# ------------------------------------------------------------------------------------------------ extra legs

FLOPS_DIT_L = 161_386_856_448   # algorithmic FLOPs per sample per NFE (SURVEY.md 8(d))
FLOPS_DIT_B = 46_003_912_704
FLOPS_UNET_CELEB512 = 189.72e9


def gemm_vs_cublas(device, iters=20):
    """The four DiT-L/2 linear layers at batch 64 (M = 16384): our wgmma kernel WITH its fused epilogue
    (bias / GELU / gated residual add) against (a) the bare torch.matmul (cuBLAS) of the same operands - `ratio` - and
    (b) the same OPERATION through the library (cuBLASLt bias epilogue + separate elementwise kernels) -
    `ratio_vs_library_same_op` - on the same box, CUDA events, alternating so that all see the same clocks.  > 1: ours is faster."""
    from lfm_b200 import _lib
    lib = _lib.load()
    s = C.c_void_p(torch.cuda.current_stream(device).cuda_stream)
    M = BATCH * 256
    out = {}
    for name, N, K, epi in (("qkv", 3072, 1024, 0), ("proj", 1024, 1024, 2), ("fc1", 4096, 1024, 1), ("fc2", 1024, 4096, 2)):
        a = torch.randn(M, K, device=device).bfloat16()
        w = (torch.randn(N, K, device=device) * 0.03).bfloat16()
        bias = torch.randn(N, device=device)
        gate = torch.randn(M // 256, N, device=device)
        o = torch.zeros(M, N, device=device, dtype=torch.float32 if epi >= 2 else torch.bfloat16)

        bn = int(os.environ.get("LFM_BENCH_GEMM_BN", "0")) or DEFAULT_GEMM_BN

        def ours():
            rc = lib.lfm_dbg_gemm(a.data_ptr(), w.data_ptr(), bias.data_ptr(), o.data_ptr(), gate.data_ptr(), N, 256, M, N, K, epi, bn, s)
            assert rc == 0, _lib.last_error()

        def cublas():
            return a @ w.t()

        bias_h = bias.bfloat16()
        xres = torch.zeros(M // 256, 256, N, device=device) if epi == 2 else None

        def library_fused():
            # the same OPERATION through the library, as an eager-PyTorch user gets it: cuBLASLt GEMM with its bias epilogue,
            # then the activation / gated residual as separate elementwise kernels
            lin = torch.nn.functional.linear(a, w, bias_h)
            if epi == 1:
                return torch.nn.functional.gelu(lin, approximate="tanh")
            if epi == 2:
                return xres.add_(gate[:, None, :] * lin.view(M // 256, 256, N))
            return lin

        def t(fn):
            for _ in range(3):
                fn()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                fn()
            e1.record()
            torch.cuda.synchronize(device)
            return e0.elapsed_time(e1) / iters * 1e3
        us_o, us_c, us_l = [], [], []
        for _ in range(3):
            us_o.append(t(ours))
            us_c.append(t(cublas))
            us_l.append(t(library_fused))
        uo, uc, ul = min(us_o), min(us_c), min(us_l)
        fl = 2.0 * M * N * K
        out[name] = {"M": M, "N": N, "K": K, "epilogue": ("bias->bf16", "bias+GELU(tanh)->bf16", "x += gate*(acc+bias), fp32")[epi],
                     "ours_us": round(uo, 1), "cublas_bare_matmul_us": round(uc, 1), "library_same_op_us": round(ul, 1),
                     "ours_tflops": round(fl / uo / 1e6, 1), "cublas_tflops": round(fl / uc / 1e6, 1),
                     "ratio": round(uc / uo, 3), "ratio_vs_library_same_op": round(ul / uo, 3)}
        del a, w, o, xres
    return out


def gpu_eager_baseline(device, nfe_run=10):
    """The reference network in eager PyTorch on THIS GPU (tests/tools/eager_dit.py): the library baseline a user of the
    reference gets on this GPU - bf16 autocast + F.scaled_dot_product_attention + TF32 on - and the reference's own
    setting, fp32 with TF32 off (test_flow_latent.py:103).  Same weights, batch and Euler grid as the headline; a bounded
    sample of nfe_run Euler steps scaled to Euler-50."""
    from tests.tools import eager_dit
    import lfm_b200
    from lfm_b200.synthetic import synthetic_state_dict
    with torch.device("meta"):
        net = lfm_b200.DiT_models[MODEL](img_resolution=32, in_channels=4, label_dropout=0.0, num_classes=1)
    sd = {k: v.to(device) for k, v in synthetic_state_dict(net, WEIGHT_SEED).items()}
    arch = dict(depth=24, hidden=1024, heads=16)
    x = torch.randn(BATCH, 4, 32, 32, device=device)
    nodes = lfm_b200.euler_time_grid(STEP_SIZE)[: nfe_run + 1].to(device)
    res = {}
    for label, tf32, ac, n in (("bf16_autocast_sdpa_tf32", True, True, nfe_run), ("fp32_tf32_off", False, False, 2)):
        torch.backends.cuda.matmul.allow_tf32 = tf32
        torch.backends.cudnn.allow_tf32 = tf32
        nd = nodes[: n + 1]
        eager_dit.euler(sd, x, nd[:2], autocast_bf16=ac, **arch)
        torch.cuda.synchronize(device)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        eager_dit.euler(sd, x, nd, autocast_bf16=ac, **arch)
        e1.record()
        torch.cuda.synchronize(device)
        ms_nfe = e0.elapsed_time(e1) / n
        res[label] = {"ms_per_nfe": round(ms_nfe, 3), "images_per_s": round(BATCH / (ms_nfe * 1e-3) / NFE, 2),
                      "tflops": round(BATCH * FLOPS_DIT_L / ms_nfe / 1e9, 1), "nfe_timed": n}
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    res["what"] = f"eager PyTorch {torch.__version__} on this GPU, DiT-L/2 batch {BATCH}, Euler NFE scaled to Euler-{NFE} images/s"
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)  # timed sampling passes, >= 1
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-extras", action="store_true", help="skip other_configs / gemm_vs_cublas / gpu_eager_baseline / decode")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write the sampled latents of the last timed step to DIR/latents.npy (float32)")
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be at least 1")
    if args.impl == "reference":
        return run_reference(args)
    if args.warmup < 3:
        args.warmup = 3

    import torch.distributed as dist
    import lfm_b200
    from lfm_b200 import dist as ldist

    if not torch.cuda.is_available():
        raise SystemExit("bench.py needs a CUDA device (H100); the lfm_b200 hot path has no CPU fallback")
    rank, world, local = ldist.init_from_env("nccl")
    if world != args.gpus and not (world == 1 and args.gpus == 1):
        if rank == 0:
            print(f"warning: --gpus {args.gpus} but WORLD_SIZE={world}", file=sys.stderr)
    device = torch.device("cuda", local)
    torch.cuda.set_device(device)
    peaks = load_peaks()
    net = build_model(device, max_batch=BATCH if args.no_extras else 128)   # 128: BASELINE.json configs[4] reuses this context
    flops_nfe = FLOPS_DIT_L
    sargs = types.SimpleNamespace(method="euler", step_size=STEP_SIZE, perturb=False, cfg_scale=1.0, compute_nfe=False)
    chw = 4 * 32 * 32

    # host-side buffers for the end-to-end leg (pinned)
    g = torch.Generator().manual_seed(ldist.rank_seed(42, rank))
    z_host = torch.randn(BATCH, 4, 32, 32, generator=g).pin_memory()
    out_host = torch.empty(BATCH, 4, 32, 32).pin_memory()
    z_dev = z_host.to(device)

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize(device)

    last = {}

    def step_device():
        xf = lfm_b200.sample_from_model(net, z_dev, {}, sargs)[-1]
        last["latents"] = ldist.all_gather_batch(xf) if world > 1 else xf
        return last["latents"]

    def step_e2e():
        z = z_host.to(device, non_blocking=True)
        xf = lfm_b200.sample_from_model(net, z, {}, sargs)[-1]
        allx = ldist.all_gather_batch(xf) if world > 1 else xf
        out_host.copy_(allx[rank::world] if world > 1 else allx, non_blocking=True)
        return allx

    def timed(fn, k, counter=None):
        """k calls of fn bracketed by barrier + synchronize; CUDA events; MAX over ranks (ms total)."""
        counter = counter or net
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        l0 = counter.launch_count()
        e0.record()
        for _ in range(k):
            fn()
        e1.record()
        barrier()
        ms = torch.tensor([e0.elapsed_time(e1)], device=device)
        if world > 1:
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return float(ms.item()), counter.launch_count() - l0

    for _ in range(args.warmup):
        step_device()
    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    ms_total, launches = timed(step_device, args.steps)
    clocks = sampler.stop() if rank == 0 else None
    if args.dump_outputs and rank == 0:
        # what a caller of the timed path receives: the Euler-50 latents of the last timed step, [BATCH * world, 4, 32, 32] (1 MB per 64)
        import numpy as np
        os.makedirs(args.dump_outputs, exist_ok=True)
        np.save(os.path.join(args.dump_outputs, "latents.npy"), last["latents"].float().cpu().numpy())
    for _ in range(2):
        step_e2e()
    ms_e2e, _ = timed(step_e2e, args.steps)

    # ------------------------------------------------------------------ BASELINE.json configs 3, 4, 5 at this GPU count
    other = {}
    decode = None
    if not args.no_extras:
        # ---- images/s INCLUDING the VAE decode (test_flow_latent.py:193): native decoder, synthetic weights, the uint8
        # post-processing fused, and the one all-gather moving the DECODED images (196 KB each) as north_star says
        from lfm_b200.vae import AutoencoderKL, synthetic_vae_state_dict
        vae = AutoencoderKL(max_batch=16)
        vae.load_state_dict(synthetic_vae_state_dict(vae, WEIGHT_SEED), strict=True)
        vae = vae.to(device).eval()

        def step_decode():
            xf = lfm_b200.sample_from_model(net, z_dev, {}, sargs)[-1]
            u8 = vae.decode_to_uint8(xf / 0.18215)
            return ldist.all_gather_batch(u8) if world > 1 else u8
        xf0 = step_device()[:BATCH].contiguous()
        step_decode()
        ms_sd, _ = timed(step_decode, 3)
        ms_sd /= 3
        fn_d = lambda: vae.decode_to_uint8(xf0 / 0.18215)  # noqa: E731
        fn_d()
        ms_d, _ = timed(fn_d, 3, vae)
        ms_d /= 3
        fl = AutoencoderKL().decode_flops_per_image(32)
        decode = {"what": f"Euler-{NFE} sampling + native AutoencoderKL decode (256x256, synthetic sd-vae-ft-mse-shaped weights) + uint8 "
                          f"post-processing, batch {BATCH}/GPU; all-gather of the decoded uint8 images for N > 1",
                  "images_per_s_with_decode": round(BATCH * world / ms_sd * 1e3, 2), "ms_per_pass": round(ms_sd, 2),
                  "decode_only_ms_per_batch": round(ms_d, 2), "decode_only_images_per_s_per_gpu": round(BATCH / ms_d * 1e3, 1),
                  "decode_tflops_per_gpu": round(BATCH * fl / ms_d / 1e9, 1), "decode_flops_per_image": fl}
        del vae
        torch.cuda.empty_cache()

        def sweep(per_gpu, nfes, reps=2):
            x = torch.randn(per_gpu, 4, 32, 32, generator=torch.Generator().manual_seed(7 + rank)).to(device)
            rows = []
            for n in nfes:
                a = types.SimpleNamespace(method="euler", step_size=1.0 / n, perturb=False, cfg_scale=1.0, compute_nfe=False)

                def fn():
                    xf = lfm_b200.sample_from_model(net, x, {}, a)[-1]
                    return ldist.all_gather_batch(xf) if world > 1 else xf
                fn()
                ms, _ = timed(fn, reps)
                ms /= reps
                rows.append({"euler_nfe": n, "images_per_s": round(per_gpu * world / ms * 1e3, 2), "ms_per_pass": round(ms, 2),
                             "tflops_per_gpu": round(n * per_gpu * FLOPS_DIT_L / ms / 1e9, 1)})
            return rows
        other["cfg5_weak"] = {"what": f"DiT-L/2 Euler NFE sweep, batch 128 per GPU (global {128 * world}), dp{world}",
                              "rows": sweep(128, (10, 20, 50, 100))}
        per = max(1, 128 // world)
        other["cfg5_strong"] = {"what": f"DiT-L/2 Euler NFE sweep, GLOBAL batch 128 => {per} per GPU (M = {per * 256} token rows), dp{world}",
                                "rows": sweep(per, (10, 20, 50, 100)) if world > 1 else "identical to cfg5_weak at 1 GPU"}
        if world == 1:
            # the per-GPU shares of the strong-scaling run (global 128 on 2 / 4 / 8 GPUs) measured on ONE GPU: what
            # strong scaling can reach is tflops(share) / tflops(128)
            rows = []
            for share, n_gpus in ((64, 2), (32, 4), (16, 8)):
                r = sweep(share, (50,))[0]
                r.update({"batch_per_gpu": share, "stands_for_n_gpus": n_gpus})
                rows.append(r)
            base = [r for r in other["cfg5_weak"]["rows"] if r["euler_nfe"] == 50][0]["tflops_per_gpu"]
            for r in rows:
                r["predicted_strong_scaling_efficiency"] = round(r["tflops_per_gpu"] / base, 3)
            other["cfg5_strong_shares_on_one_gpu"] = {"what": "Euler-50 at the per-GPU batch of a global-128 run on 2 / 4 / 8 GPUs, one GPU",
                                                      "rows": rows}
    del net
    torch.cuda.empty_cache()
    if not args.no_extras:
        # cfg3: DiT-B/2, 1000 classes, CFG 1.5, Karras Heun-25 (48 NFE, 2 network rows per image), 32 images per GPU
        nb = build_model(device, "DiT-B/2", 1000, 0.1, 64)
        gg = torch.Generator().manual_seed(11 + rank)
        xb = torch.randn(32, 4, 32, 32, generator=gg).to(device)
        yb = torch.randint(0, 1000, (32,), generator=gg).to(device)
        mk = dict(y=torch.cat([yb, torch.full((32,), 1000, device=device)]), cfg_scale=1.5)

        def fn3():
            out = lfm_b200.karras_sample(nb, torch.cat([xb, xb]), 25, clip_denoised=False, model_kwargs=mk, sigma_min=1e-5,
                                         sigma_max=1.0, sampler="heun")[:32]
            return ldist.all_gather_batch(out) if world > 1 else out
        fn3()
        ms, _ = timed(fn3, 3, nb)
        ms /= 3
        nfe3 = nb.last_stats["nfe"]
        other["cfg3"] = {"what": f"DiT-B/2 imnet, CFG 1.5, Heun-25 ({nfe3} NFE x 2 rows), 32 images per GPU (global {32 * world}), dp{world}",
                         "images_per_s": round(32 * world / ms * 1e3, 2), "ms_per_pass": round(ms, 2),
                         "tflops_per_gpu": round(nfe3 * 64 * FLOPS_DIT_B / ms / 1e9, 1)}
        del nb
        torch.cuda.empty_cache()
        if world == 1:
            # cfg4: ADM UNetModel celeb512 (64x64x4 latents), dopri5 atol = rtol = 1e-5, batch 32, one GPU
            nu = build_unet_celeb512(device, 32)
            xu = torch.randn(32, 4, 64, 64, generator=torch.Generator().manual_seed(13)).to(device)
            a4 = types.SimpleNamespace(method="dopri5", atol=1e-5, rtol=1e-5, cfg_scale=1.0, compute_nfe=True)
            fn4 = lambda: lfm_b200.sample_from_model(nu, xu, {}, a4)  # noqa: E731
            fn4()
            ms, _ = timed(fn4, 2, nu)
            ms /= 2
            st = nu.last_stats
            other["cfg4"] = {"what": "ADM UNetModel celeb512 preset, dopri5 atol=rtol=1e-5, batch 32, 1 GPU", **st,
                             "images_per_s": round(32 / ms * 1e3, 2), "ms_per_pass": round(ms, 2),
                             "tflops_per_gpu": round(st["nfe"] * 32 * FLOPS_UNET_CELEB512 / ms / 1e9, 1)}
            del nu
            torch.cuda.empty_cache()
            # Not BASELINE configurations: the two DiT geometries outside (256 tokens, head_dim 64) - DiT-XL/2 (head_dim 72) and DiT-L/2 on
            # 64 x 64 latents (1024 tokens, 512-pixel images) - whose attention runs on the mma.sync flash kernel.  Euler-10, one GPU.
            for key, model, side, per_gpu in (("dit_xl2", "DiT-XL/2", 32, 64), ("dit_l2_64x64_latents", "DiT-L/2", 64, 16)):
                ng = build_model(device, model, 1, 0.0, per_gpu, latent_side=side)
                xg = torch.randn(per_gpu, 4, side, side, generator=torch.Generator().manual_seed(17)).to(device)
                ag = types.SimpleNamespace(method="euler", step_size=0.1, perturb=False, cfg_scale=1.0, compute_nfe=False)
                fng = lambda: lfm_b200.sample_from_model(ng, xg, {}, ag)[-1]  # noqa: E731
                fng()
                ms, _ = timed(fng, 2, ng)
                ms /= 2
                T_, D_, L_ = (side // 2) ** 2, ng.hidden_size, ng.depth
                fl = L_ * (24 * T_ * D_ * D_ + 4 * T_ * T_ * D_ + 12 * D_ * D_) + 4 * T_ * 16 * D_ + 2 * (256 * D_ + D_ * D_) + 4 * D_ * D_
                other[key] = {"what": f"{model} on {side}x{side} latents ({T_} tokens, head_dim {D_ // ng.num_heads}), Euler-10, batch {per_gpu}, 1 GPU",
                              "images_per_s": round(per_gpu / ms * 1e3, 2), "ms_per_pass": round(ms, 2),
                              "tflops_per_gpu": round(10 * per_gpu * fl / ms / 1e9, 1), "flops_per_sample_per_nfe": fl}
                del ng
                torch.cuda.empty_cache()

    if rank == 0:
        imgs = BATCH * world * args.steps
        value = imgs / (ms_total * 1e-3)
        e2e_value = imgs / (ms_e2e * 1e-3)
        tflops = value * NFE * flops_nfe / 1e12 / world  # per GPU
        extras = {}
        if world == 1 and not args.no_extras:
            extras["gpu_eager_baseline"] = gpu_eager_baseline(device)
            extras["gemm_vs_cublas"] = gemm_vs_cublas(device)
        cpu = None
        if world == 1 and not args.no_cpu_baseline:
            threads = usable_threads()
            v, dt, sample = cpu_baseline(threads)
            cpu = {"value": round(v, 5), "unit": "images/s", "cores": threads, "kind": "port", "sample": sample}
        elif world == 1:
            time.sleep(3.0)
        # the dominant kernel is timed ALONE against the burst peak: the CPU leg above (or the pause) lets the board
        # leave the power-capped state of the long run first, as in the measurement of the burst peak itself
        roof = time_dominant_kernel(device, peaks) if world == 1 else None
        line = {
            "metric": "images/sec DiT-L/2 32x32 latents Euler-50", "value": round(value, 3), "unit": "images/s",
            "n_gpus": world, "steps": args.steps, "warmup": args.warmup, "ms_per_step": round(ms_total / args.steps, 3),
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "bf16", "data": "synthetic",
            "config": workload_config(world),
            "nfe_img_per_s": round(value * NFE, 1),
            "e2e": {"value": round(e2e_value, 3), "unit": "images/s", "h2d_bytes_per_step": BATCH * chw * 4,
                    "d2h_bytes_per_step": BATCH * chw * 4, "ms_per_step": round(ms_e2e / args.steps, 3)},
            "gpu_launches": int(launches),
            "clocks": clocks,
            "roofline_forward": {"bound": "tensor", "achieved": round(tflops, 1), "unit": "TFLOP/s per GPU",
                                 "peak_sustained": peaks["sustained"], "frac_sustained": round(tflops / peaks["sustained"], 4),
                                 "peak_burst": peaks["burst"], "frac_burst": round(tflops / peaks["burst"], 4),
                                 "flops_per_sample_per_nfe": flops_nfe, "peak_source": peaks["source"]},
        }
        if roof is not None:
            line["roofline"] = roof
        if cpu is not None:
            line["cpu_baseline"] = cpu
        if decode is not None:
            line["decode"] = decode
        if other:
            line["other_configs"] = other
        line.update(extras)
        print(json.dumps(line), flush=True)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
