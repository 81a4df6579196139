"""Concat-conditioned UNetModel (the downstream tasks' WrapperCondFlow, model(t, cat([x, cond], 1))) on the H100.

  * conv_in, the only kernel the conditioning changes: every output against an fp64 reference on the same fp32 operands, within
    (K + 16) 2^-23 (|x| * |w| + |bias|) with K = 9 Cin (DESIGN.md section 4), for one and two sources;
  * one NFE of the 9- and 8-channel mini networks against fixtures of the reference's own module (scripts/make_cond_goldens.py);
  * every native solver with a stored condition against the oracle, and the condition buffer refreshed under the cached graphs;
  * the unconditioned networks bit-identical to the bytes recorded before conv_in was generalised (scripts/make_unet_golden.py).
"""
import ctypes as C
import importlib.util
import os
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import lfm_b200
from lfm_b200 import _lib
from oracle import solvers as osol
from oracle import unet as ounet
from tests._util import T, load_golden, rel_l2

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL_UNET_NFE = 1e-2   # the ADM bound of tests/test_gpu_parity.py


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


def P(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


# ------------------------------------------------------------------------------------------------ conv_in kernel

def run_conv_in(a, b, w, bias, side, a_stride=None, b_stride=None):
    B, Cout = a.shape[0], w.shape[0]
    out = torch.empty(B, side, side, Cout, device=a.device)
    a_ch = a.shape[1] if a_stride is None else w.shape[1] - (b.shape[1] if b is not None else 0)
    b_ch = 0 if b is None else w.shape[1] - a_ch
    a_st = a_stride if a_stride is not None else a_ch * side * side
    b_st = b_stride if b_stride is not None else b_ch * side * side
    _lib.check(_lib.load().lfm_dbg_conv_in(P(a), a_ch, a_st, P(b), b_ch, b_st, P(w), P(bias), P(out), B, side, Cout, None))
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("side", [4, 12, 16, 32, 64, 256])   # 4 and 12: conv_in_kernel; multiples of 8: the strip kernel
@pytest.mark.parametrize("cin,b_ch", [(3, 0), (4, 0), (8, 0), (9, 0), (8, 4), (9, 5), (4, 1)])
def test_conv_in_vs_fp64(dev, side, cin, b_ch):
    g = torch.Generator().manual_seed(side * 31 + cin * 7 + b_ch)
    B, Cout = 2, 128 if side < 256 else 64
    x = torch.randn(B, cin, side, side, generator=g)
    w = torch.randn(Cout, cin, 3, 3, generator=g) / 3
    bias = torch.randn(Cout, generator=g)
    a, b = x[:, :cin - b_ch].contiguous(), (x[:, cin - b_ch:].contiguous() if b_ch else None)
    out = run_conv_in(a.to(dev), b.to(dev) if b is not None else None, w.to(dev), bias.to(dev), side).cpu().double()
    ref = F.conv2d(x.double(), w.double(), bias.double(), padding=1).permute(0, 2, 3, 1)
    mag = F.conv2d(x.double().abs(), w.double().abs(), bias.double().abs(), padding=1).permute(0, 2, 3, 1)
    bound = (9 * cin + 16) * 2.0 ** -23 * mag
    assert ((out - ref).abs() <= bound).all(), float(((out - ref).abs() / mag).max())


def test_conv_in_reads_slices_of_one_tensor(dev):
    """lfm_forward's layout: both sources are channel slices of one [B, 9, H, W] tensor (image stride 9 H W)."""
    g = torch.Generator().manual_seed(5)
    x = torch.randn(3, 9, 32, 32, generator=g)
    w = torch.randn(128, 9, 3, 3, generator=g) / 3
    bias = torch.randn(128, generator=g)
    xd = x.to(dev)
    hw = 32 * 32
    out = run_conv_in(xd, xd[:, 4:], w.to(dev), bias.to(dev), 32, a_stride=9 * hw, b_stride=9 * hw)
    two = run_conv_in(x[:, :4].contiguous().to(dev), x[:, 4:].contiguous().to(dev), w.to(dev), bias.to(dev), 32)
    assert torch.equal(out, two)


# ------------------------------------------------------------------------------------------------ networks

def cfg_from_golden(g):
    return ounet.UNetConfig(image_size=int(g["cfg_image_size"]), in_channels=int(g["cfg_in_channels"]),
                            model_channels=int(g["cfg_model_channels"]), out_channels=int(g["cfg_out_channels"]),
                            num_res_blocks=int(g["cfg_num_res_blocks"]),
                            attention_resolutions=tuple(int(v) for v in g["cfg_attention_resolutions"]),
                            channel_mult=tuple(int(v) for v in g["cfg_channel_mult"]), num_heads=int(g["cfg_num_heads"]),
                            num_head_channels=int(g["cfg_num_head_channels"]))


def make_net(cfg, sd, dev, max_batch=None):
    net = lfm_b200.UNetModel(image_size=cfg.image_size, in_channels=cfg.in_channels, model_channels=cfg.model_channels,
                             out_channels=4, num_res_blocks=cfg.num_res_blocks, attention_resolutions=cfg.attention_resolutions,
                             channel_mult=cfg.channel_mult, num_heads=cfg.num_heads, num_head_channels=cfg.num_head_channels,
                             use_scale_shift_norm=True, max_batch=max_batch)
    net.load_state_dict(sd, strict=True)
    return net.to(dev).eval()


def setup(name, dev):
    g = load_golden(name)
    cfg = cfg_from_golden(g)
    sd = ounet.synthetic_state_dict(cfg, int(g["weight_seed"]))
    return g, cfg, sd, make_net(cfg, sd, dev)


@pytest.mark.parametrize("name", ["unet_inpaint_mini", "unet_semantic_mini"])
def test_conditioned_forward_vs_reference_fixture(dev, name):
    g, cfg, sd, net = setup(name, dev)
    z, cond = T(g["z"]).to(dev), T(g["cond"]).to(dev)
    wrapped = lfm_b200.WrapperCondFlow(net, cond)
    v = wrapped(T(g["t_vec"]).to(dev), z)
    assert v.shape == z.shape
    assert rel_l2(v.cpu(), g["v"]) < TOL_UNET_NFE
    # the condition is read: another condition gives another velocity
    v2 = lfm_b200.WrapperCondFlow(net, cond.flip(0))(T(g["t_vec"]).to(dev), z)
    assert rel_l2(v2.cpu(), v.cpu()) > 1e-2
    # lfm_forward(cat[z, c]) is the velocity of the sampler's first Euler stage (t = 1): x1 = z + (0 - 1) v  for one step
    v1 = wrapped(torch.tensor(1.0, device=dev), z)
    args = types.SimpleNamespace(method="euler", step_size=1.0, perturb=False, atol=1e-5, rtol=1e-5)
    x1 = lfm_b200.downstream.sample_from_model(wrapped, z, args)[-1]
    assert torch.equal(x1, z - v1)
    with pytest.raises(ValueError):
        net(0.5, z)                                                   # 4 channels into a 9- / 8-channel network


@pytest.mark.parametrize("name", ["unet_inpaint_mini", "unet_semantic_mini"])
def test_conditioned_fixed_step_solvers(dev, name):
    g, cfg, sd, net = setup(name, dev)
    z, cond = T(g["z"]), T(g["cond"])
    wrapped = lfm_b200.WrapperCondFlow(net, cond.to(dev))
    h = float(g["euler_step"])
    f = lambda t, x: ounet.unet_forward(sd, cfg, t, torch.cat([x, cond], 1))  # noqa: E731
    for m in ("euler", "midpoint", "rk4"):
        args = types.SimpleNamespace(method=m, step_size=h, perturb=False, atol=1e-5, rtol=1e-5)
        traj = lfm_b200.downstream.sample_from_model(wrapped, z.to(dev), args)
        ref = T(g["euler"]) if m == "euler" else osol.tdq_fixed_rk(f, z, h, m)[0]
        assert rel_l2(traj[-1].cpu(), ref) < 2e-2, m
        assert wrapped.count_nfe is True


@pytest.mark.parametrize("method", ["dopri5", "bosh3", "adaptive_heun"])
def test_conditioned_adaptive_solvers(dev, method):
    g, cfg, sd, net = setup("unet_inpaint_mini", dev)
    z, cond = T(g["z"]), T(g["cond"])
    wrapped = lfm_b200.WrapperCondFlow(net, cond.to(dev))
    args = types.SimpleNamespace(method=method, atol=1e-3, rtol=1e-3, compute_fid=True)
    traj = lfm_b200.downstream.sample_from_model(wrapped, z.to(dev), args)
    nfe = net.last_stats["nfe"]
    fb = lambda t, x: ounet.unet_forward(sd, cfg, t, torch.cat([x, cond], 1), emulate_bf16=True)  # noqa: E731
    refb, st = osol.tdq_adaptive(fb, z, method=method, rtol=1e-3, atol=1e-3)
    assert rel_l2(traj[-1].cpu(), refb) < 2e-2
    assert abs(nfe - st.nfe) <= 12, (nfe, st.nfe)


def test_condition_refreshed_under_cached_graphs(dev):
    g, cfg, sd, net = setup("unet_semantic_mini", dev)
    z, cond = T(g["z"]).to(dev), T(g["cond"]).to(dev)
    conds = [cond, torch.randn(cond.shape, generator=torch.Generator().manual_seed(3)).to(dev)]
    for m, extra in (("rk4", dict(step_size=0.25, perturb=False)), ("dopri5", dict())):
        args = types.SimpleNamespace(method=m, atol=1e-3, rtol=1e-3, **extra)
        same_ctx = [lfm_b200.downstream.sample_from_model(lfm_b200.WrapperCondFlow(net, c), z, args)[-1] for c in conds]
        for c, got in zip(conds, same_ctx):
            fresh = make_net(cfg, sd, dev)
            assert torch.equal(got, lfm_b200.downstream.sample_from_model(lfm_b200.WrapperCondFlow(fresh, c), z, args)[-1])
        assert not torch.equal(same_ctx[0], same_ctx[1])


def test_conditioned_sampler_refusals(dev):
    g, cfg, sd, net = setup("unet_inpaint_mini", dev)
    z, cond = T(g["z"]).to(dev), T(g["cond"]).to(dev)
    args = types.SimpleNamespace(method="euler", step_size=0.5, perturb=False, atol=1e-5, rtol=1e-5)
    with pytest.raises(ValueError):                                   # no condition on the chain
        lfm_b200.downstream.sample_from_model(net, z, args)
    with pytest.raises(ValueError):                                   # a condition for another batch
        lfm_b200.downstream.sample_from_model(lfm_b200.WrapperCondFlow(net, cond[:1]), z, args)
    lib = _lib.load()
    ctx = net.native(2, dev)
    assert lib.lfm_set_condition(ctx, P(cond), 2, 4, None) != 0 and "channels" in _lib.last_error(ctx)
    assert lib.lfm_set_condition(ctx, P(cond), 3, 5, None) != 0 and "B_img" in _lib.last_error(ctx)
    _lib.check(lib.lfm_set_condition(ctx, P(cond), 1, 5, None), ctx)
    x = z.clone()
    grid = torch.tensor([1.0, 0.5, 0.0])
    stats = _lib.OdeStats()
    assert lib.lfm_sample_fixed(ctx, 0, P(x), P(grid), 3, 0, 0, None, 2, 1.0, C.byref(stats), None) != 0
    assert "lfm_set_condition" in _lib.last_error(ctx)
    with pytest.raises(NotImplementedError):
        lfm_b200.downstream.sample_from_model(lfm_b200.WrapperCondFlow(net, cond), z,
                                              types.SimpleNamespace(method="dopri8", atol=1e-5, rtol=1e-5))


# ------------------------------------------------------------------------------------------------ unchanged bytes

def load_recipe():
    spec = importlib.util.spec_from_file_location("make_unet_golden", os.path.join(ROOT, "scripts", "make_unet_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_unet_and_edm_bit_identical_to_the_recorded_fingerprint(dev):
    """The UNetModel forwards (4-channel, class-conditional) and a celeb512 dopri5 trajectory, and the DhariwalUNet forwards (without
    and with labels, forward_with_cfg) and a CFG Euler run, give the bytes recorded by scripts/make_unet_golden.py
    (tests/golden/unet_fingerprint.npz)."""
    g = np.load(os.path.join(ROOT, "tests", "golden", "unet_fingerprint.npz"))
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if int(g["num_sms"]) != sms:
        pytest.skip(f"fingerprint recorded with {int(g['num_sms'])} SMs ({g['device']}); the split-K plan differs on {sms}")
    got = load_recipe().fingerprint(dev)
    assert sorted(got) == sorted(k for k in g.files if k.endswith(("_sha256", "_sub")))
    for k, v in got.items():
        if k.endswith("_sub"):
            assert np.array_equal(v, g[k]), k
        else:
            assert v == str(g[k]), k
