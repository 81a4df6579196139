"""Reference-facing ODE solver entry points, executed by liblfm_b200.so.

Same names, arguments and return shapes as the reference:

* ``sample_from_model(model, x_0, model_kwargs, args)``                      test_flow_latent.py:42-76
* ``sample_from_model_with_fixed_step_solver(model, x, model_kwargs, generator, args)``   test_flow_latent.py:79-97
* ``karras_sample(model, x_T, steps, ...)`` with ``sampler in {"euler", "heun"}``  sampler/karras_sample.py:7-76

The time grids are built here exactly as the reference's dependencies build them (fp32 ``linspace`` for the
Karras samplers; torchdiffeq's ``arange * step_size + t0`` for ``--method euler``) and handed to the native
sampler, which integrates the whole trajectory on the device from a captured CUDA graph - no per-step Python,
no host synchronisation.  Configurations the native path does not implement raise ``NotImplementedError``;
nothing silently falls back to PyTorch.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib
from .network import _NativeNet

ADAPTIVE_SOLVER = ["dopri5", "dopri8", "adaptive_heun", "bosh3"]   # test_flow_latent.py:27
FIXER_SOLVER = ["euler", "rk4", "midpoint", "stochastic"]         # test_flow_latent.py:28

# sampler/karras_sample.py:129,155: sample_heun's corrector guard is `i < steps - 1` with the function
# default steps=40, which karras_sample never overrides => intervals >= 39 are Euler-only.
HEUN_REFERENCE_CORRECTOR_LIMIT = 39


def _unwrap(model):
    """Accept the NFECount-style wrappers of the reference CLI and the downstream tasks' WrapperCondFlow (attribute .model;
    _condition reads the latter's .cond)."""
    inner = model
    while not isinstance(inner, _NativeNet) and hasattr(inner, "model"):
        inner = inner.model
    if not isinstance(inner, _NativeNet):
        raise TypeError("lfm_b200 solvers need an lfm_b200 network (got %r)" % type(model).__name__)
    return inner


def _condition(model):
    """The condition a chain of WrapperCondFlow-style wrappers (attribute .cond) concatenates to the state: the wrapper
    nearest the caller concatenates first, so the network sees cat([x, cond_outer, ..., cond_inner], 1).  None without one."""
    conds = []
    inner = model
    while not isinstance(inner, _NativeNet) and hasattr(inner, "model"):
        if getattr(inner, "cond", None) is not None:
            conds.append(inner.cond)
        inner = inner.model
    return torch.cat(conds, 1) if conds else None


def _set_condition(net, ctx, cond, x):
    """Hand the wrapper chain's condition to a concat-conditioned network (lfm_set_condition) before a native sampler runs."""
    n_cond = net.in_channels - net.out_channels
    if cond is None:
        if n_cond:
            raise ValueError(f"the network takes {net.in_channels} input channels: wrap it in WrapperCondFlow(model, cond) with "
                             f"a {n_cond}-channel condition")
        return
    if cond.dim() != 4 or cond.shape[0] != x.shape[0] or cond.shape[2:] != x.shape[2:] or cond.shape[1] != n_cond:
        raise ValueError(f"the condition must be [{x.shape[0]}, {n_cond}, {x.shape[2]}, {x.shape[3]}] for this network and state "
                         f"(got {tuple(cond.shape)})")
    cond = cond.to(device=x.device, dtype=torch.float32).contiguous()
    _lib.check(_lib.load().lfm_set_condition(ctx, cond.data_ptr(), x.shape[0], n_cond, _NativeNet._stream(x.device)), ctx)


def _split_cfg(x, model_kwargs):
    """The reference evolves the doubled batch [x, x] with labels [y, y_null] (test_flow_latent.py:171-181);
    both halves stay identical, so the native sampler evolves one copy and evaluates 2B network rows per NFE."""
    cfg_scale = float(model_kwargs.get("cfg_scale", 1.0)) if model_kwargs else 1.0
    y = model_kwargs.get("y") if model_kwargs else None
    if cfg_scale > 1.0:
        if x.shape[0] % 2:
            raise ValueError("cfg_scale > 1 expects the doubled batch [x, x]")
        n = x.shape[0] // 2
        if y is None:
            raise ValueError("cfg_scale > 1 needs labels")
        return x[:n].contiguous(), y, cfg_scale, True
    return x.contiguous(), y, 1.0, False


def _check_labels(net, y, rows, device):
    """Label validation shared by every sampler entry (the same checks ``forward`` applies in ``_prep``): one label
    per network row, each a valid row of the network's label table - the reference's ``nn.Embedding`` /
    ``F.one_hot`` raise on an out-of-range label, and the C ABI reads exactly ``rows`` labels from the pointer."""
    if y is None or not net.uses_labels():
        return None
    y = torch.as_tensor(y, device=device).to(torch.int64).reshape(-1).contiguous()
    if y.numel() != rows:
        raise ValueError(f"expected {rows} labels, got {y.numel()}")
    net.check_label_range(y)
    return y


def _run_native(model, x, y, cfg_scale, entry, method, *args):
    """Integrate a float32 copy of x with the native sampler ``entry`` (lfm_sample_fixed or lfm_sample_adaptive), called
    as ``entry(ctx, method, x, *args, y, B_img, cfg_scale, stats, stream)``.  Returns (x_final, stats dict)."""
    net = _unwrap(model)
    if not x.is_cuda:
        raise RuntimeError("lfm_b200 solvers run on CUDA tensors only")
    x = x.to(torch.float32).contiguous().clone()
    n_img = x.shape[0]
    rows = 2 * n_img if cfg_scale > 1.0 else n_img
    y = _check_labels(net, y, rows, x.device)
    ctx = net.native(rows, x.device)
    _set_condition(net, ctx, _condition(model), x)
    stats = _lib.OdeStats()
    _lib.check(getattr(_lib.load(), entry)(
        ctx, method, x.data_ptr(), *args, y.data_ptr() if y is not None else None, n_img, float(cfg_scale), C.byref(stats),
        _NativeNet._stream(x.device)), ctx)
    net.last_stats = dict(nfe=int(stats.nfe), accepted=int(stats.accepted), rejected=int(stats.rejected))
    return x, net.last_stats


def _run_fixed(model, x, y, cfg_scale, t_nodes, method, t_as_vector, corrector_limit):
    grid = t_nodes.detach().to("cpu", torch.float32).contiguous()
    return _run_native(model, x, y, cfg_scale, "lfm_sample_fixed", {"euler": 0, "heun": 1, "midpoint": 2, "rk4": 3}[method],
                       grid.data_ptr(), grid.numel(), int(t_as_vector), int(corrector_limit))


def euler_time_grid(step_size: float, t0: float = 1.0, t1: float = 0.0) -> torch.Tensor:
    """Model-time nodes of torchdiffeq's fixed-grid solvers for t = [t0, t1], t0 > t1 (time is negated
    internally: s = -t; grid s_k = arange(niters) * step_size + s_0 in fp32, niters = ceil((s_1 - s_0) / h + 1),
    last node forced to s_1)."""
    s = -torch.tensor([t0, t1], dtype=torch.float32)
    niters = int(torch.ceil((s[-1] - s[0]) / step_size + 1).item())
    grid = torch.arange(0, niters, dtype=torch.float32) * step_size + s[0]
    grid[-1] = s[-1]
    return -grid


def sample_from_model(model, x_0, model_kwargs, args):
    """test_flow_latent.py:42-76: ``odeint(denoiser, x_0, t=[1, 0], method=args.method, ...)``.
    Returns the [2, B, C, H, W] trajectory (x_0, x_final); with ``args.compute_nfe`` also the NFE count."""
    method = args.method
    mk = dict(model_kwargs or {})
    # the reference's denoiser picks forward_with_cfg from args.cfg_scale and forwards **model_kwargs, whose
    # cfg_scale entry is the scale actually applied (test_flow_latent.py:55-59, 171-181)
    if float(getattr(args, "cfg_scale", 1.0)) > 1.0:
        mk.setdefault("cfg_scale", float(args.cfg_scale))
    else:
        mk.pop("cfg_scale", None)
    x, y, cfg_scale, doubled = _split_cfg(x_0, mk)
    if method in ("euler", "midpoint", "rk4"):
        flags = 2 if getattr(args, "perturb", False) else 0        # LFM_FIXED_PERTURB (test_flow_latent.py:44-48,64)
        nodes = euler_time_grid(float(args.step_size))
        xf, stats = _run_fixed(model, x, y, cfg_scale, nodes, method, flags, 0)
    elif method in ("dopri5", "bosh3", "adaptive_heun"):
        xf, stats = _run_native(model, x, y, cfg_scale, "lfm_sample_adaptive", {"dopri5": 0, "bosh3": 1, "adaptive_heun": 2}[method],
                                1.0, 0.0, float(args.rtol), float(args.atol))
    else:
        raise NotImplementedError(f"method '{method}' has no native implementation (euler, midpoint, rk4, dopri5, bosh3 and "
                                  "adaptive_heun do)")
    if doubled:
        xf = torch.cat([xf, xf], 0)
    traj = torch.stack([x_0.to(xf.dtype), xf], 0)
    if getattr(args, "compute_nfe", False):
        return traj, torch.tensor(float(stats["nfe"]), device=xf.device)
    return traj


def karras_sample(model, x_T, steps, clip_denoised=True, progress=False, callback=None, model_kwargs=None, device=None,
                  sigma_min=0.002, sigma_max=80, sampler="heun", s_churn=0.0, s_tmin=0.0, s_tmax=float("inf"),
                  s_noise=1.0, generator=None, classifier=None, cond_func=None, heun_corrector_limit=None,
                  consume_rng=True, **unused):
    """sampler/karras_sample.py:7-76.  ``rho`` / ``ts`` (passed by the reference CLI, which the reference's own
    function rejects) are accepted and ignored."""
    if sampler not in ("euler", "heun"):
        raise KeyError(sampler)
    if clip_denoised or classifier is not None or callback is not None or s_churn != 0.0:
        raise NotImplementedError("native karras_sample supports clip_denoised=False, s_churn=0, no classifier/callback "
                                  "(the configuration test_flow_latent.py:79-97 uses)")
    sigmas = torch.linspace(sigma_max, sigma_min, steps, device="cpu", dtype=torch.float32)
    x, y, cfg_scale, doubled = _split_cfg(x_T, model_kwargs or {})
    limit = HEUN_REFERENCE_CORRECTOR_LIMIT if heun_corrector_limit is None else int(heun_corrector_limit)
    if sampler == "heun" and consume_rng and generator is not None:
        # sample_heun draws generator.randn_like(x) once per interval and multiplies it by 0
        # (karras_sample.py:145); consume the same random numbers so that later batches see the same RNG state.
        for _ in range(steps - 1):
            generator.randn_like(x_T)
    xf, _ = _run_fixed(model, x, y, cfg_scale, sigmas, sampler, 1, limit)
    if doubled:
        xf = torch.cat([xf, xf], 0)
    return xf


def sample_from_model_with_fixed_step_solver(model, x, model_kwargs, generator, args):
    """test_flow_latent.py:79-97 (with the reference's unsupported rho/ts kwargs dropped)."""
    return karras_sample(model, x, steps=args.num_steps, model_kwargs=model_kwargs, device=x.device, clip_denoised=False,
                         sigma_min=1e-5, sigma_max=1.0, s_tmin=0.0, s_tmax=1.0, s_churn=0.0, sampler=args.method,
                         generator=generator)


# the misspelt name test_flow_latent.py:188 calls
sample_from_model_with_fixed_step_solve = sample_from_model_with_fixed_step_solver
