"""Parity tests proper (H100 only, `-m gpu`): the CUDA path, called through the C ABI (liblfm_b200.so via
lfm_b200's ctypes binding), against the CPU oracle, the committed reference fixtures, and size-independent
properties at BASELINE.json's full sizes.

Tolerances (the reference pins none; SURVEY.md 8(d)).  The CUDA path keeps the residual stream, LayerNorm
statistics, softmax, adaLN parameters, the ODE state and time in fp32 and rounds only tensor-core operands and
the stored qkv / attention / MLP-hidden activations to bf16:
  * one network evaluation vs the fp32 reference fixture .......... rel-L2 <= 2e-3   (measured ~1.2e-4)
  * end-to-end sampler output vs the fp32 reference fixture ....... rel-L2 <= 2e-3   (measured ~3e-5)
  * solver arithmetic given identical velocities .................. bit-exact / <= 1e-6
  * kernel-level GEMM vs fp32 matmul of the same bf16 operands .... fp32 out <= 1e-5, bf16 out <= 4e-3 (1 bf16 ulp)
"""
import ctypes as C
import types

import pytest
import torch

import lfm_b200
from lfm_b200 import _lib
from oracle import dit as odit
from oracle import solvers as osol
from tests._util import T, cfg_from_golden, load_golden, oracle_model, rel_l2

pytestmark = pytest.mark.gpu

TOL_NFE = 2e-3
TOL_E2E = 2e-3


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


def P(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def make_net(cfg, sd, dev, max_batch=None):
    net = lfm_b200.DiT(img_resolution=cfg.img_resolution, patch_size=cfg.patch_size, in_channels=cfg.in_channels,
                       hidden_size=cfg.hidden_size, depth=cfg.depth, num_heads=cfg.num_heads,
                       label_dropout=cfg.label_dropout, num_classes=cfg.num_classes, max_batch=max_batch)
    net.load_state_dict(sd, strict=True)
    return net.to(dev).eval()


def make_big(model_type, dev, num_classes, label_dropout, max_batch):
    from lfm_b200.synthetic import synthetic_state_dict
    with torch.device("meta"):
        net = lfm_b200.DiT_models[model_type](img_resolution=32, in_channels=4, label_dropout=label_dropout,
                                              num_classes=num_classes, max_batch=max_batch)
    sd = synthetic_state_dict(net, 1)
    net = net.to_empty(device="cpu")
    net.load_state_dict(sd, strict=True)
    return net.to(dev).eval()


# ------------------------------------------------------------------------------------------------ kernels


@pytest.mark.parametrize("M,N,K,epi,bn", [
    (128, 128, 64, 3, 128), (256, 512, 1024, 0, 256), (512, 1024, 1024, 1, 256), (512, 1024, 4096, 2, 256),
    (512, 1024, 4096, 2, 128), (64, 2048, 1024, 3, 256), (4, 1024, 256, 3, 256), (256, 1152, 384, 0, 256),
    (256, 1152, 384, 1, 128), (16384, 3072, 1024, 0, 256), (16384, 1024, 1024, 2, 128),
    # block_n 512 / 1024 / 640: the tile width the network picks for the shape (128 x 256, or 128 x 128 when the launch is tile-starved),
    # incl. N tails and M tails
    (256, 256, 64, 3, 512), (768, 1152, 384, 0, 512), (512, 1024, 4096, 2, 512), (16384, 1024, 4096, 2, 512),
    (16384, 3072, 1024, 1, 512), (768, 768, 384, 1, 1024), (512, 1024, 4096, 2, 1024), (16384, 3072, 1024, 0, 1024),
    (512, 256, 64, 3, 640), (256, 256, 128, 3, 640), (768, 1152, 384, 0, 640), (1280, 768, 256, 1, 640), (512, 1024, 4096, 2, 640),
    (4096, 1024, 1024, 2, 640), (16384, 1024, 4096, 2, 640), (16384, 3072, 1024, 1, 640), (16384, 4096, 1024, 0, 640),
    (32768, 1024, 1024, 2, 640), (38 * 512, 512, 128, 3, 640)])
def test_gemm_epilogues(dev, M, N, K, epi, bn):
    lib = _lib.load()
    g = torch.Generator().manual_seed(M + N + K + epi)
    a = (torch.randn(M, K, generator=g) * 0.5).to(dev).bfloat16()
    w = (torch.randn(N, K, generator=g) * 0.05).to(dev).bfloat16()
    bias = torch.randn(N, generator=g).to(dev)
    Tt = 256
    gate = torch.randn((M + Tt - 1) // Tt, 3 * N, generator=g).to(dev)
    acc = a.float() @ w.float().t() + bias
    if epi == 0:
        out, ref, tol = torch.zeros(M, N, device=dev, dtype=torch.bfloat16), acc, 4e-3
    elif epi == 1:
        out, ref, tol = (torch.zeros(M, N, device=dev, dtype=torch.bfloat16),
                         torch.nn.functional.gelu(acc, approximate="tanh"), 4e-3)
    elif epi == 2:
        x0 = torch.randn(M, N, generator=g).to(dev)
        out = x0.clone()
        ref = x0 + gate[torch.arange(M, device=dev) // Tt, N:2 * N] * acc
        tol = 1e-5
    else:
        out, ref, tol = torch.zeros(M, N, device=dev), acc, 1e-5
    rc = lib.lfm_dbg_gemm(P(a), P(w), P(bias), P(out), C.c_void_p(gate.data_ptr() + N * 4), 3 * N, Tt, M, N, K, epi, bn,
                          None)
    torch.cuda.synchronize()
    assert rc == 0, _lib.last_error()
    assert rel_l2(out.float().cpu(), ref.cpu()) < tol


@pytest.mark.parametrize("variant", [0, 1])   # 0: TMA + wgmma kernel (the network's), 1: mma.sync flash kernel on the same layout
@pytest.mark.parametrize("B,H", [(1, 1), (2, 4), (3, 12), (64, 16), (5, 16), (7, 6), (33, 12), (128, 16)])
def test_attention(dev, variant, B, H):
    lib = _lib.load()
    D = H * 64
    g = torch.Generator().manual_seed(B * 100 + H)
    qkv = torch.randn(B * 256, 3 * D, generator=g).to(dev).bfloat16()
    q, k, v = qkv.float().reshape(B, 256, 3, H, 64).permute(2, 0, 3, 1, 4)
    ref = (torch.softmax((q @ k.transpose(-1, -2)) * 0.125, dim=-1) @ v).transpose(1, 2).reshape(B * 256, D)
    out = torch.zeros(B * 256, D, device=dev, dtype=torch.bfloat16)
    rc = lib.lfm_dbg_attention(P(qkv), P(out), B, H, variant, None, None)
    torch.cuda.synchronize()
    assert rc == 0, _lib.last_error()
    assert rel_l2(out.float().cpu(), ref.cpu()) < 5e-3   # P and O are rounded to bf16


@pytest.mark.parametrize("B,H,T,ch,dh", [(2, 4, 1024, 64, 64), (3, 16, 256, 80, 72), (2, 3, 256, 64, 64), (5, 16, 64, 80, 72),
                                         (7, 16, 16, 80, 72), (1, 2, 128, 80, 72)])
def test_attention_mma_kernels(dev, B, H, T, ch, dh):
    """The mma.sync attention kernels of the DiT geometries outside T = 256 / head_dim 64 (head-major qkv rows, heads zero-padded from dh
    to ch channels) against softmax(q k^T / sqrt(dh)) v in fp32 on the same bf16 operands."""
    lib = _lib.load()
    g = torch.Generator().manual_seed(B * 1000 + T + ch)
    qkv = torch.randn(B, T, H, 3, ch, generator=g)
    qkv[..., dh:] = 0                                            # the padding channels are zero (zero weight rows)
    qkv = qkv.reshape(B * T, H * 3 * ch).to(dev).bfloat16()
    q, k, v = qkv.float().reshape(B, T, H, 3, ch).permute(3, 0, 2, 1, 4)    # [B, H, T, ch] each
    ref = (torch.softmax((q @ k.transpose(-1, -2)) * dh ** -0.5, dim=-1) @ v).transpose(1, 2).reshape(B * T, H * ch)
    out = torch.full((B * T, H * ch), 7.0, device=dev, dtype=torch.bfloat16)
    rc = lib.lfm_dbg_attention_mma(P(qkv), P(out), B, H, T, ch, dh, None)
    torch.cuda.synchronize()
    assert rc == 0, _lib.last_error()
    assert rel_l2(out.float().cpu(), ref.cpu()) < 5e-3           # P and O are rounded to bf16
    if ch > dh:
        assert float(out.float().reshape(B * T, H, ch)[..., dh:].abs().max()) == 0.0   # padded output channels are exactly zero


# ------------------------------------------------------------------------------------------------ reference fixtures


# patch 4 / 8 and other latent sides: token grids 8 x 8 / 4 x 4 (short-sequence attention kernel on head-major qkv rows, generic
# patch-embed / final-layer kernels) and 16 x 16 with patch 4 on 64 x 64 latents (oracle/make_goldens.py patch)
GEOMETRY = ["mini_p4", "mini_p8", "mini_r64p4", "mini_r16p2",
            # head_dim 72 (the DiT-XL width: heads stored padded to 80 channels) at 256 / 64 tokens; 1024 tokens (64 x 64 latents, /2)
            "mini_xl2", "mini_xl4", "mini_r64p2"]


@pytest.mark.parametrize("name", ["mini_uncond", "mini_cond", "mini_d384"] + GEOMETRY)
def test_forward_vs_reference_fixture(dev, name):
    g = load_golden(name)
    cfg = cfg_from_golden(g)
    net = make_net(cfg, odit.synthetic_state_dict(cfg, int(g["weight_seed"])), dev)
    x = T(g["x"]).to(dev)
    v = net(T(g["t_scalar"]).to(dev), x)                       # 0-d t, y=None
    assert rel_l2(v.cpu(), g["v_scalar_ynone"]) < TOL_NFE
    v = net(T(g["t_vec"]).to(dev), x, T(g["y"]).to(dev))       # [B] t, labels
    assert rel_l2(v.cpu(), g["v_vec_y"]) < TOL_NFE
    v = net(float(g["t_scalar"]), x)                           # python float t
    assert rel_l2(v.cpu(), g["v_scalar_ynone"]) < TOL_NFE
    if cfg.num_classes > 1:
        x2 = torch.cat([x, x])
        v = net.forward_with_cfg(torch.full((4,), 0.4, device=dev), x2, T(g["y_cfg"]).to(dev), cfg_scale=1.5)
        assert rel_l2(v.cpu(), g["v_cfg_1p5"]) < TOL_NFE
        assert torch.equal(v[:2], v[2:])
        with pytest.raises(IndexError):
            net(0.5, x, torch.tensor([0, cfg.num_classes + 5], device=dev))


@pytest.mark.parametrize("name", ["mini_uncond", "mini_cond", "mini_d384"] + GEOMETRY)
def test_fixed_step_samplers_vs_reference_fixture(dev, name):
    g = load_golden(name)
    cfg = cfg_from_golden(g)
    net = make_net(cfg, odit.synthetic_state_dict(cfg, int(g["weight_seed"])), dev)
    x = T(g["x"]).to(dev)
    if cfg.num_classes > 1:
        xs, mk = torch.cat([x, x]), dict(y=T(g["y_cfg"]).to(dev), cfg_scale=1.5)
    else:
        xs, mk = x, {}
    kw = dict(clip_denoised=False, model_kwargs=mk, sigma_min=1e-5, sigma_max=1.0)
    out = lfm_b200.karras_sample(net, xs, 6, sampler="euler", **kw)
    assert rel_l2(out.cpu(), g["euler6"]) < TOL_E2E and net.last_stats["nfe"] == 5
    out = lfm_b200.karras_sample(net, xs, 5, sampler="heun", **kw)
    assert rel_l2(out.cpu(), g["heun5"]) < TOL_E2E and net.last_stats["nfe"] == 8
    args = types.SimpleNamespace(num_steps=6, method="euler")
    out2 = lfm_b200.sample_from_model_with_fixed_step_solver(net, xs, mk, None, args)
    assert rel_l2(out2.cpu(), g["euler6"]) < TOL_E2E


def test_heun_reference_quirk(dev):
    g = load_golden("mini_uncond")
    cfg = cfg_from_golden(g)
    net = make_net(cfg, odit.synthetic_state_dict(cfg, int(g["weight_seed"])), dev)
    x = T(g["x"]).to(dev)
    kw = dict(clip_denoised=False, model_kwargs={}, sigma_min=1e-5, sigma_max=1.0, sampler="heun")
    out = lfm_b200.karras_sample(net, x, 43, **kw)
    assert rel_l2(out.cpu(), g["heun43"]) < TOL_E2E
    assert net.last_stats["nfe"] == 2 * 39 + 3                  # intervals 39..41 are Euler-only
    out = lfm_b200.karras_sample(net, x, 43, heun_corrector_limit=10 ** 6, **kw)
    assert net.last_stats["nfe"] == 84


def test_full_size_dit_l2_fixture(dev):
    g = load_golden("dit_l2")
    net = make_big("DiT-L/2", dev, 1, 0.0, 2)
    x = T(g["x"]).to(dev)
    v = net(T(g["t"]).to(dev), x)
    assert rel_l2(v.cpu(), g["v"]) < TOL_NFE
    out = lfm_b200.karras_sample(net, x, 3, clip_denoised=False, model_kwargs={}, sigma_min=1e-5, sigma_max=1.0,
                                 sampler="euler")
    assert rel_l2(out.cpu(), g["euler3"]) < TOL_E2E


def test_full_size_dit_b2_cfg_fixture(dev):
    g = load_golden("dit_b2")
    net = make_big("DiT-B/2", dev, 1000, 0.1, 4)
    x = T(g["x"]).to(dev)
    v = net.forward_with_cfg(T(g["t"]).to(dev), torch.cat([x, x]), T(g["y_cfg"]).to(dev), cfg_scale=1.5)
    assert rel_l2(v.cpu(), g["v_cfg_1p5"]) < TOL_NFE


# ------------------------------------------------------------------------------------------------ torchdiffeq paths vs oracle


def test_torchdiffeq_euler_and_dopri5_vs_oracle(dev):
    g = load_golden("mini_uncond")
    cfg = cfg_from_golden(g)
    sd = odit.synthetic_state_dict(cfg, int(g["weight_seed"]))
    net = make_net(cfg, sd, dev)
    x = T(g["x"])
    f = oracle_model(sd, cfg)
    args = types.SimpleNamespace(method="euler", step_size=0.1, perturb=False, cfg_scale=1.0, compute_nfe=True)
    traj, nfe = lfm_b200.sample_from_model(net, x.to(dev), {}, args)
    ref, n = osol.tdq_euler(f, x, 0.1)
    assert traj.shape == (2, 2, 4, 32, 32) and int(nfe) == n == 10
    assert torch.equal(traj[0].cpu(), x)
    assert rel_l2(traj[-1].cpu(), ref) < TOL_E2E
    args = types.SimpleNamespace(method="dopri5", atol=1e-5, rtol=1e-5, cfg_scale=1.0, compute_nfe=True)
    traj, nfe = lfm_b200.sample_from_model(net, x.to(dev), {}, args)
    ref, st = osol.tdq_dopri5(f, x)
    assert rel_l2(traj[-1].cpu(), ref) < TOL_E2E
    s = net.last_stats
    assert s["nfe"] == 2 + 6 * (s["accepted"] + s["rejected"]) == int(nfe)
    # bf16 noise in v perturbs the embedded error estimate at rtol 1e-5: step counts may differ by a step or two
    assert abs(s["nfe"] - st.nfe) <= 12
    # at a tolerance well above the bf16 noise floor the accept/reject sequence must agree exactly
    args = types.SimpleNamespace(method="dopri5", atol=1e-2, rtol=1e-2, cfg_scale=1.0, compute_nfe=True)
    traj, nfe = lfm_b200.sample_from_model(net, x.to(dev), {}, args)
    ref, st = osol.tdq_dopri5(f, x, rtol=1e-2, atol=1e-2)
    assert (net.last_stats["nfe"], net.last_stats["accepted"], net.last_stats["rejected"]) == (st.nfe, st.accepted, st.rejected)
    assert rel_l2(traj[-1].cpu(), ref) < TOL_E2E
    for m, per in (("midpoint", 2), ("rk4", 4)):
        args = types.SimpleNamespace(method=m, step_size=0.2, perturb=False, cfg_scale=1.0, compute_nfe=True)
        traj, nfe = lfm_b200.sample_from_model(net, x.to(dev), {}, args)
        ref, n = osol.tdq_fixed_rk(f, x, 0.2, m)
        assert int(nfe) == n == 5 * per
        assert rel_l2(traj[-1].cpu(), ref) < TOL_E2E
    # options["perturb"] (--perturb, test_flow_latent.py:44-48,64): first evaluation of a step one ulp past the node
    for m in ("euler", "rk4"):
        args = types.SimpleNamespace(method=m, step_size=0.2, perturb=True, cfg_scale=1.0, compute_nfe=False)
        traj = lfm_b200.sample_from_model(net, x.to(dev), {}, args)
        ref = (osol.tdq_euler(f, x, 0.2, perturb=True) if m == "euler" else osol.tdq_fixed_rk(f, x, 0.2, m, perturb=True))[0]
        assert rel_l2(traj[-1].cpu(), ref) < TOL_E2E
    # the other adaptive pairs of torchdiffeq the CLI accepts (test_flow_latent.py:27): same controller, other tableau
    for m, per in (("bosh3", 3), ("adaptive_heun", 1)):
        args = types.SimpleNamespace(method=m, atol=1e-2, rtol=1e-2, cfg_scale=1.0, compute_nfe=True)
        traj, nfe = lfm_b200.sample_from_model(net, x.to(dev), {}, args)
        ref, st = osol.tdq_adaptive(f, x, m, rtol=1e-2, atol=1e-2)
        s = net.last_stats
        assert (s["nfe"], s["accepted"], s["rejected"]) == (st.nfe, st.accepted, st.rejected) and int(nfe) == 2 + per * (st.accepted + st.rejected)
        assert rel_l2(traj[-1].cpu(), ref) < TOL_E2E
        args = types.SimpleNamespace(method=m, atol=1e-3, rtol=1e-3, cfg_scale=1.0, compute_nfe=False)
        traj = lfm_b200.sample_from_model(net, x.to(dev), {}, args)
        ref, st = osol.tdq_adaptive(f, x, m, rtol=1e-3, atol=1e-3)
        assert rel_l2(traj[-1].cpu(), ref) < TOL_E2E and abs(net.last_stats["nfe"] - st.nfe) <= 6 * per
    with pytest.raises(NotImplementedError):
        lfm_b200.sample_from_model(net, x.to(dev), {}, types.SimpleNamespace(method="dopri8", step_size=0.1, cfg_scale=1.0, atol=1e-3, rtol=1e-3))


def test_dopri5_with_cfg_vs_oracle(dev):
    g = load_golden("mini_cond")
    cfg = cfg_from_golden(g)
    sd = odit.synthetic_state_dict(cfg, int(g["weight_seed"]))
    net = make_net(cfg, sd, dev)
    x = T(g["x"])
    y2 = T(g["y_cfg"])
    args = types.SimpleNamespace(method="dopri5", atol=1e-3, rtol=1e-3, cfg_scale=1.5, compute_nfe=False)
    traj = lfm_b200.sample_from_model(net, torch.cat([x, x]).to(dev), dict(y=y2.to(dev), cfg_scale=1.5), args)
    ref, st = osol.tdq_dopri5(oracle_model(sd, cfg, y2, 1.5), torch.cat([x, x]), rtol=1e-3, atol=1e-3)
    assert traj.shape[1] == 4 and torch.equal(traj[-1][:2], traj[-1][2:])
    assert rel_l2(traj[-1].cpu(), ref) < TOL_E2E
    # accept/reject decisions can flip by one step under bf16 noise in v; the solution must still agree
    assert abs(net.last_stats["nfe"] - st.nfe) <= 6 and net.last_stats["nfe"] == 2 + 6 * (
        net.last_stats["accepted"] + net.last_stats["rejected"])


# ------------------------------------------------------------------------------------------------ full-size properties


@pytest.fixture(scope="module")
def dit_l2_b64(dev):
    return make_big("DiT-L/2", dev, 1, 0.0, 64)


def test_full_size_properties_dit_l2_b64(dev, dit_l2_b64):
    """BASELINE.json configs[1] size (DiT-L/2, batch 64): properties that need no full-size oracle run."""
    net = dit_l2_b64
    g = torch.Generator().manual_seed(5)
    x = torch.randn(64, 4, 32, 32, generator=g).to(dev)
    t = torch.tensor(0.6, device=dev)
    v1 = net(t, x)
    v2 = net(t, x)
    assert torch.equal(v1, v2)                                   # deterministic / idempotent
    assert torch.isfinite(v1).all() and float(v1.abs().mean()) > 1e-3
    # samples are independent: any sub-batch gives the same rows (same kernels, same per-row arithmetic)
    v_half = net(t, x[16:48])
    assert rel_l2(v_half.cpu(), v1[16:48].cpu()) < 1e-6
    perm = torch.randperm(64, generator=g).to(dev)
    assert rel_l2(net(t, x[perm]).cpu(), v1[perm].cpu()) < 1e-6
    # a [B] vector of equal times == a 0-d time (models/DiT.py:65-66 broadcast)
    assert torch.equal(net(torch.full((64,), 0.6, device=dev), x), v1)
    # spot-check 2 rows of the batch against the fp32 oracle
    from lfm_b200.synthetic import synthetic_state_dict
    cfg = odit.make_config("DiT-L/2", num_classes=1, label_dropout=0.0)
    sd = {k: v.detach().cpu() for k, v in net.state_dict().items()}
    ref = odit.dit_forward(sd, cfg, torch.tensor(0.6), x[[3, 60]].cpu())
    assert rel_l2(v1[[3, 60]].cpu(), ref) < TOL_NFE
    # one Euler interval == x + dt * v   (solver arithmetic is exact fp32)
    nodes = torch.tensor([0.6, 0.35])
    args = types.SimpleNamespace(method="euler", step_size=0.02, perturb=False, cfg_scale=1.0, compute_nfe=False)
    from lfm_b200 import solvers
    xf, st = solvers._run_fixed(net, x, None, 1.0, nodes, "euler", 0, 0)
    assert torch.equal(xf, x + v1 * (nodes[1] - nodes[0]).item()) or rel_l2(xf.cpu(), (x + v1 * (nodes[1] - nodes[0]).to(dev)).cpu()) < 1e-7
    # Euler-50 end to end: finite, moved, and two half-batches reproduce the full batch
    full = lfm_b200.sample_from_model(net, x, {}, args)[-1]
    assert net.last_stats["nfe"] == 50 and torch.isfinite(full).all()
    halves = torch.cat([lfm_b200.sample_from_model(net, x[:32], {}, args)[-1],
                        lfm_b200.sample_from_model(net, x[32:], {}, args)[-1]])
    assert rel_l2(halves.cpu(), full.cpu()) < 1e-5
    assert float((full - x).abs().mean()) > 1e-2


def test_cfg_identity_dit_b2_full(dev):
    """configs[2] shape (DiT-B/2, 32 images x2 under CFG): forward_with_cfg == u + s (c - u) of two plain forwards."""
    net = make_big("DiT-B/2", dev, 1000, 0.1, 64)
    g = torch.Generator().manual_seed(9)
    x = torch.randn(32, 4, 32, 32, generator=g).to(dev)
    y = torch.randint(0, 1000, (32,), generator=g).to(dev)
    ynull = torch.full((32,), 1000, device=dev)
    t = torch.full((64,), 0.45, device=dev)
    v = net.forward_with_cfg(t, torch.cat([x, x]), torch.cat([y, ynull]), cfg_scale=1.5)
    c = net(t[:32], x, y)
    u = net(t[:32], x, ynull)
    assert rel_l2(v[:32].cpu(), (u + 1.5 * (c - u)).cpu()) < 1e-5
    assert torch.equal(v[:32], v[32:])
    # y=None selects the null class row (models/DiT.py:259-260)
    assert torch.equal(net(t[:32], x), u)
    # Heun-25 with CFG (configs[2] solver): 48 NFE, finite
    out = lfm_b200.karras_sample(net, torch.cat([x, x]), 25, clip_denoised=False,
                                 model_kwargs=dict(y=torch.cat([y, ynull]), cfg_scale=1.5), sigma_min=1e-5, sigma_max=1.0,
                                 sampler="heun")
    assert net.last_stats["nfe"] == 48 and torch.isfinite(out).all() and torch.equal(out[:32], out[32:])


# ------------------------------------------------------------------------------------------------ ADM UNetModel

TOL_UNET_NFE = 1e-2   # ~60 bf16-operand convolutions per evaluation (measured 5.5e-3); SURVEY.md 8(d)


def make_unet(cfg, sd, dev, max_batch=None):
    net = lfm_b200.UNetModel(image_size=cfg.image_size, in_channels=4, model_channels=cfg.model_channels, out_channels=4,
                             num_res_blocks=cfg.num_res_blocks, attention_resolutions=cfg.attention_resolutions,
                             channel_mult=cfg.channel_mult, num_classes=cfg.num_classes, num_heads=cfg.num_heads,
                             num_head_channels=cfg.num_head_channels, use_scale_shift_norm=True, max_batch=max_batch)
    net.load_state_dict(sd, strict=True)
    return net.to(dev).eval()


@pytest.mark.parametrize("name", ["unet_mini", "unet_mini_cond", "unet_celeb256"])
def test_unet_forward_vs_reference_fixture(dev, name):
    from oracle import unet as ounet
    from tests.test_oracle_unet import unet_cfg_from_golden
    g = load_golden(name)
    cfg = unet_cfg_from_golden(g) if name != "unet_celeb256" else ounet.UNetConfig(image_size=32, channel_mult=(1, 2, 2, 2))
    net = make_unet(cfg, ounet.synthetic_state_dict(cfg, int(g["weight_seed"])), dev)
    x = T(g["x"]).to(dev)
    y = T(g["y"]).to(dev) if "y" in g else None
    v = net(T(g["t_vec"]).to(dev), x, y)
    assert rel_l2(v.cpu(), g["v"]) < TOL_UNET_NFE
    assert torch.equal(v, net(T(g["t_vec"]).to(dev), x, y))            # deterministic
    if y is None:
        with pytest.raises(AssertionError):
            net(0.5, x, torch.zeros(x.shape[0], dtype=torch.long, device=dev))   # unet.py:622-624
        # a sub-batch reproduces its rows (odd batch sizes exercise the partial 128-pixel tiles)
        v1 = net(T(g["t_vec"])[:1].to(dev), x[:1])
        assert rel_l2(v1.cpu(), v[:1].cpu()) < 1e-5
    else:
        with pytest.raises(AssertionError):
            net(0.5, x)
        with pytest.raises(RuntimeError):
            net.native(x.shape[0], x.device)
            lfm_b200.karras_sample(net, torch.cat([x, x]), 3, clip_denoised=False, sampler="euler", sigma_min=1e-5,
                                   sigma_max=1.0, model_kwargs=dict(y=torch.cat([y, y]), cfg_scale=1.5))


def test_unet_solvers_vs_oracle(dev):
    from oracle import unet as ounet
    from tests.test_oracle_unet import unet_cfg_from_golden
    g = load_golden("unet_mini")
    cfg = unet_cfg_from_golden(g)
    sd = ounet.synthetic_state_dict(cfg, int(g["weight_seed"]))
    net = make_unet(cfg, sd, dev)
    x = T(g["x"])
    f = lambda tt, xx: ounet.unet_forward(sd, cfg, tt, xx)  # noqa: E731
    out = lfm_b200.karras_sample(net, x.to(dev), 4, clip_denoised=False, model_kwargs={}, sigma_min=1e-5, sigma_max=1.0,
                                 sampler="heun")
    assert rel_l2(out.cpu(), osol.karras_sample(f, x, 4, "heun")) < TOL_UNET_NFE and net.last_stats["nfe"] == 6
    args = types.SimpleNamespace(method="dopri5", atol=1e-2, rtol=1e-2, cfg_scale=1.0, compute_nfe=True)
    traj, nfe = lfm_b200.sample_from_model(net, x.to(dev), {}, args)
    ref, st = osol.tdq_dopri5(f, x, rtol=1e-2, atol=1e-2)
    assert rel_l2(traj[-1].cpu(), ref) < TOL_UNET_NFE
    assert abs(int(nfe) - st.nfe) <= 6 and int(nfe) == 2 + 6 * (net.last_stats["accepted"] + net.last_stats["rejected"])
    args = types.SimpleNamespace(method="euler", step_size=0.25, perturb=False, cfg_scale=1.0, compute_nfe=False)
    traj = lfm_b200.sample_from_model(net, x.to(dev), {}, args)
    assert rel_l2(traj[-1].cpu(), osol.tdq_euler(f, x, 0.25)[0]) < TOL_UNET_NFE


def test_unet_celeb512_full_size_properties(dev):
    """BASELINE.json configs[3] network (celeb512 preset, 64x64x4 latents): batch-independence, finiteness, one
    oracle spot check, and a dopri5 run with a loose tolerance (NFE accounting)."""
    from lfm_b200.synthetic import synthetic_unet_state_dict
    from oracle import unet as ounet
    with torch.device("meta"):
        net = lfm_b200.UNetModel(image_size=64, in_channels=4, model_channels=256, out_channels=4, num_res_blocks=2,
                                 attention_resolutions=(16, 8), channel_mult=(1, 2, 2, 2, 4), num_heads=4,
                                 use_scale_shift_norm=True, max_batch=8)
    sd = synthetic_unet_state_dict(net, 1)
    assert len(sd) == 396
    net = net.to_empty(device="cpu")
    net.load_state_dict(sd, strict=True)
    net = net.to(dev).eval()
    g = torch.Generator().manual_seed(2)
    x = torch.randn(8, 4, 64, 64, generator=g).to(dev)
    v = net(torch.tensor(0.5, device=dev), x)
    assert torch.isfinite(v).all() and float(v.abs().mean()) > 1e-2
    assert rel_l2(net(0.5, x[2:5]).cpu(), v[2:5].cpu()) < 1e-5
    ref = ounet.unet_forward(sd, ounet.UNetConfig(), torch.tensor(0.5), x[:1].cpu())
    assert rel_l2(v[:1].cpu(), ref) < TOL_UNET_NFE
    args = types.SimpleNamespace(method="dopri5", atol=5e-2, rtol=5e-2, cfg_scale=1.0, compute_nfe=True)
    traj, nfe = lfm_b200.sample_from_model(net, x, {}, args)
    s = net.last_stats
    assert int(nfe) == 2 + 6 * (s["accepted"] + s["rejected"]) and torch.isfinite(traj[-1]).all()


def test_cfg4_unet_celeb512_batch32_dopri5_1e5(dev):
    """BASELINE.json configs[3] AS STATED: UNetModel celeb512 preset (test_args/celeb512_adm.txt), batch 32, dopri5 with
    atol = rtol = 1e-5 (test_flow_latent.py:61-73, 376-377).  The native context is finalised for 32 rows (the
    split-K / tile decisions of the bench configuration) and stays the same for every call below:
      * one NFE at batch 32: two rows of the batch against the fp32 oracle;
      * dopri5 1e-5 on 2 latents (what the CPU oracle integrates in about a minute) against oracle.unet +
        oracle.solvers.tdq_dopri5: x_final vs the fp32 oracle (SURVEY.md 8(d): rel-L2 <= 2e-2), and the NFE count vs the
        oracle network evaluated WITH bf16 operand rounding.  Why: at rtol = 1e-5 the embedded error estimate
        dt * sum_j c_err,j k_j is dominated by the rounding noise of the bf16-operand convolutions (measured 5e-3 rel.
        per evaluation on this network), so the bf16 path is forced to ~3x smaller steps than an fp32 evaluation of the
        same smooth synthetic field (the native path needs several times the NFE of the fp32 oracle).  That is a property of
        bf16 compute under an adaptive solver, not of the solver code: with the same noise floor in the oracle the step
        counts agree to within two steps, and the fixed points (x_final) agree either way;
      * dopri5 1e-5 at the full batch 32: accounting, finiteness, and the batch-wide error norm at work (the step
        sequence of 32 latents differs from that of 2)."""
    from lfm_b200.synthetic import synthetic_unet_state_dict
    from oracle import unet as ounet
    with torch.device("meta"):
        net = lfm_b200.UNetModel(image_size=64, in_channels=4, model_channels=256, out_channels=4, num_res_blocks=2,
                                 attention_resolutions=(16, 8), channel_mult=(1, 2, 2, 2, 4), num_heads=4,
                                 use_scale_shift_norm=True, max_batch=32)
    sd = synthetic_unet_state_dict(net, 1)
    net = net.to_empty(device="cpu")
    net.load_state_dict(sd, strict=True)
    net = net.to(dev).eval()
    cfg = ounet.UNetConfig()
    g = torch.Generator().manual_seed(4)
    x = torch.randn(32, 4, 64, 64, generator=g)
    v = net(torch.tensor(0.7, device=dev), x.to(dev))
    assert torch.isfinite(v).all()
    ref = ounet.unet_forward(sd, cfg, torch.tensor(0.7), x[[5, 29]])
    assert rel_l2(v[[5, 29]].cpu(), ref) < TOL_UNET_NFE
    f = lambda tt, xx: ounet.unet_forward(sd, cfg, tt, xx)  # noqa: E731
    args = types.SimpleNamespace(method="dopri5", atol=1e-5, rtol=1e-5, cfg_scale=1.0, compute_nfe=True)
    traj, nfe = lfm_b200.sample_from_model(net, x[:2].to(dev), {}, args)
    s = dict(net.last_stats)
    ref, st = osol.tdq_dopri5(f, x[:2], rtol=1e-5, atol=1e-5)
    assert int(nfe) == s["nfe"] == 2 + 6 * (s["accepted"] + s["rejected"])
    assert rel_l2(traj[-1].cpu(), ref) < 2e-2
    assert s["nfe"] >= st.nfe                                     # bf16 noise can only cost steps
    fb = lambda tt, xx: ounet.unet_forward(sd, cfg, tt, xx, emulate_bf16=True)  # noqa: E731
    refb, stb = osol.tdq_dopri5(fb, x[:2], rtol=1e-5, atol=1e-5)
    assert abs(s["nfe"] - stb.nfe) <= 12, (s, stb.nfe, st.nfe)
    assert rel_l2(traj[-1].cpu(), refb) < 2e-2
    traj, nfe = lfm_b200.sample_from_model(net, x.to(dev), {}, args)
    s32 = net.last_stats
    assert int(nfe) == 2 + 6 * (s32["accepted"] + s32["rejected"]) and torch.isfinite(traj[-1]).all()
    assert 20 <= s32["nfe"] <= 400 and float((traj[-1] - traj[0]).abs().mean()) > 1e-2


# ------------------------------------------------------------------------------------------------ EDM DhariwalUNet


def make_edm(cfg, sd, dev, max_batch=None):
    net = lfm_b200.DhariwalUNet(img_resolution=cfg.img_resolution, in_channels=4, out_channels=4, label_dim=cfg.label_dim,
                                model_channels=cfg.model_channels, channel_mult=cfg.channel_mult, num_blocks=cfg.num_blocks,
                                attn_resolutions=cfg.attn_resolutions, dropout=0.0, max_batch=max_batch)
    net.load_state_dict(sd, strict=True)
    return net.to(dev).eval()


@pytest.mark.parametrize("name", ["edm_mini", "edm_mini_cond", "edm_ffhq", "edm_attn32"])
def test_edm_forward_vs_reference_fixture(dev, name):
    """DhariwalUNet (models/EDM.py) through lfm_create_edm vs outputs of the reference's own module: vector and 0-d t,
    labels, forward_with_cfg (drop_half_label), both attention kernels (256-token flash mma.sync / short-grid SIMT), the
    resampling blocks and the 56-channel groups of the 1792-wide concatenation (edm_ffhq)."""
    from oracle import edm as oedm
    from tests.test_oracle_edm import edm_cfg_from_golden
    g = load_golden(name)
    cfg = edm_cfg_from_golden(g)
    net = make_edm(cfg, oedm.synthetic_state_dict(cfg, int(g["weight_seed"])), dev)
    x = T(g["x"]).to(dev)
    y = T(g["y"]).to(dev) if "y" in g else None
    v = net(T(g["t_vec"]).to(dev), x, y)
    assert rel_l2(v.cpu(), g["v"]) < TOL_UNET_NFE
    assert torch.equal(v, net(T(g["t_vec"]).to(dev), x, y))            # deterministic
    assert rel_l2(net(T(g["t_scalar"]).to(dev), x).cpu(), g["v_scalar"]) < TOL_UNET_NFE   # 0-d t, y = None
    v1 = net(T(g["t_vec"])[:1].to(dev), x[:1], y[:1] if y is not None else None)
    assert rel_l2(v1.cpu(), v[:1].cpu()) < 1e-5
    if y is None:
        # without map_label a y argument is ignored (EDM.py:823)
        assert torch.equal(net(T(g["t_vec"]).to(dev), x, torch.zeros(x.shape[0], dtype=torch.long, device=dev)), v)
    else:
        x2 = torch.cat([x, x], 0)
        vc = net.forward_with_cfg(T(g["t_cfg"]).to(dev), x2, T(g["y_cfg"]).to(dev), cfg_scale=1.25)
        assert rel_l2(vc.cpu(), g["v_cfg_1p25"]) < TOL_UNET_NFE
        n = x.shape[0]
        assert torch.equal(vc[:n], vc[n:])
        # the labels of the second half are dropped whatever they are
        y_other = torch.cat([T(g["y_cfg"])[:n], torch.full((n,), cfg.label_dim - 1)]).to(dev)
        assert torch.equal(net.forward_with_cfg(T(g["t_cfg"]).to(dev), x2, y_other, cfg_scale=1.25), vc)
        with pytest.raises(RuntimeError):
            net(0.5, x, torch.full((n,), cfg.label_dim, device=dev))   # one_hot rejects class ids >= label_dim


def test_edm_solvers_vs_oracle(dev):
    """The solver entry points on a DhariwalUNet: Karras Heun with CFG (imnet_adm style: y_null = zeros, CFG 1.25),
    torchdiffeq-grid Euler and dopri5."""
    from oracle import edm as oedm
    from tests.test_oracle_edm import edm_cfg_from_golden
    g = load_golden("edm_mini_cond")
    cfg = edm_cfg_from_golden(g)
    sd = oedm.synthetic_state_dict(cfg, int(g["weight_seed"]))
    net = make_edm(cfg, sd, dev)
    x = T(g["x"])[:2]
    y = T(g["y"])[:2]
    y2 = torch.cat([y, torch.zeros_like(y)])
    fc = lambda tt, xx: oedm.edm_forward_with_cfg(sd, cfg, tt, xx, y2, 1.25)  # noqa: E731
    out = lfm_b200.karras_sample(net, torch.cat([x, x]).to(dev), 4, clip_denoised=False, sigma_min=1e-5, sigma_max=1.0,
                                 sampler="heun", model_kwargs=dict(y=y2.to(dev), cfg_scale=1.25))
    assert rel_l2(out.cpu(), osol.karras_sample(fc, torch.cat([x, x]), 4, "heun")) < TOL_UNET_NFE
    assert net.last_stats["nfe"] == 6 and torch.equal(out[:2], out[2:])
    # the same entry point against the reference's OWN karras_sample on its own DhariwalUNet (fixtures recorded by
    # oracle/make_goldens.py: Euler / Heun through the reference's CFG denoiser dispatch, and labels without CFG)
    xg, yg2 = T(g["x"]), T(g["y_cfg"])
    common = dict(clip_denoised=False, sigma_min=1e-5, sigma_max=1.0)
    out = lfm_b200.karras_sample(net, torch.cat([xg, xg]).to(dev), 4, sampler="euler", model_kwargs=dict(y=yg2.to(dev), cfg_scale=1.25), **common)
    assert rel_l2(out.cpu(), g["cfg_euler4"]) < TOL_UNET_NFE
    out = lfm_b200.karras_sample(net, torch.cat([xg, xg]).to(dev), 3, sampler="heun", model_kwargs=dict(y=yg2.to(dev), cfg_scale=1.25), **common)
    assert rel_l2(out.cpu(), g["cfg_heun3"]) < TOL_UNET_NFE
    out = lfm_b200.karras_sample(net, xg.to(dev), 3, sampler="euler", model_kwargs=dict(y=T(g["y"]).to(dev)), **common)
    assert rel_l2(out.cpu(), g["y_euler3"]) < TOL_UNET_NFE
    f = lambda tt, xx: oedm.edm_forward(sd, cfg, tt, xx, y)  # noqa: E731
    args = types.SimpleNamespace(method="euler", step_size=0.25, perturb=False, cfg_scale=1.0, compute_nfe=False)
    traj = lfm_b200.sample_from_model(net, x.to(dev), dict(y=y.to(dev)), args)
    assert rel_l2(traj[-1].cpu(), osol.tdq_euler(f, x, 0.25)[0]) < TOL_UNET_NFE
    args = types.SimpleNamespace(method="dopri5", atol=1e-2, rtol=1e-2, cfg_scale=1.0, compute_nfe=True)
    traj, nfe = lfm_b200.sample_from_model(net, x.to(dev), dict(y=y.to(dev)), args)
    ref, st = osol.tdq_dopri5(f, x, rtol=1e-2, atol=1e-2)
    assert rel_l2(traj[-1].cpu(), ref) < TOL_UNET_NFE
    assert abs(int(nfe) - st.nfe) <= 6 and int(nfe) == 2 + 6 * (net.last_stats["accepted"] + net.last_stats["rejected"])


def test_edm_imnet_preset_full_size_properties(dev):
    """The imnet_adm preset (test_args/imnet_adm.txt: nf 256, ch_mult 1 2 3 4, attention at 16 / 8 / 4, 1000 classes)
    at batch 8: finiteness, batch independence, CFG halves, one oracle spot check."""
    from lfm_b200.synthetic import synthetic_edm_state_dict
    from oracle import edm as oedm
    with torch.device("meta"):
        net = lfm_b200.DhariwalUNet(img_resolution=32, in_channels=4, out_channels=4, label_dim=1000, model_channels=256,
                                    channel_mult=(1, 2, 3, 4), num_blocks=2, attn_resolutions=(16, 8, 4), max_batch=16)
    sd = synthetic_edm_state_dict(net, 1)
    net = net.to_empty(device="cpu")
    net.load_state_dict(sd, strict=True)
    net = net.to(dev).eval()
    g = torch.Generator().manual_seed(3)
    x = torch.randn(8, 4, 32, 32, generator=g)
    y = torch.randint(0, 1000, (8,), generator=g)
    v = net(torch.tensor(0.5, device=dev), x.to(dev), y.to(dev))
    assert torch.isfinite(v).all() and float(v.abs().mean()) > 1e-2
    assert rel_l2(net(0.5, x[2:5].to(dev), y[2:5].to(dev)).cpu(), v[2:5].cpu()) < 1e-5
    cfg = oedm.EDMConfig(label_dim=1000)
    ref = oedm.edm_forward(sd, cfg, torch.tensor(0.5), x[:1], y[:1])
    assert rel_l2(v[:1].cpu(), ref) < TOL_UNET_NFE
    vc = net.forward_with_cfg(torch.tensor(0.5, device=dev), torch.cat([x, x]).to(dev), torch.cat([y, torch.zeros_like(y)]).to(dev),
                              cfg_scale=1.25)
    vu = net(torch.tensor(0.5, device=dev), x.to(dev))                   # y = None: the label term is skipped
    assert rel_l2(vc[:8].cpu(), (vu + 1.25 * (v - vu)).cpu()) < 1e-4


def test_edm_unsupported_configuration_fails_loudly(dev):
    """Self-attention on a 64x64 grid (4096 tokens) has no native kernel: lfm_create_edm must refuse (and release the
    half-built context), never fall back; a supported network created afterwards works."""
    net = lfm_b200.DhariwalUNet(img_resolution=64, in_channels=4, out_channels=4, model_channels=128, channel_mult=(1, 2),
                                num_blocks=1, attn_resolutions=(64,)).to(dev)
    with pytest.raises(RuntimeError, match="not supported"):
        net(torch.tensor(0.5, device=dev), torch.randn(1, 4, 64, 64, device=dev))
    ok = lfm_b200.DhariwalUNet(img_resolution=16, in_channels=4, out_channels=4, model_channels=128, channel_mult=(1, 2),
                               num_blocks=1, attn_resolutions=(8,)).to(dev)
    v = ok(torch.tensor(0.5, device=dev), torch.randn(2, 4, 16, 16, device=dev))
    assert v.shape == (2, 4, 16, 16) and float(v.abs().max()) == 0.0     # reference init: zero output convolution


# ------------------------------------------------------------------------------------------------ VAE decode

# ~30 bf16-operand convolutions + one attention per decode.  With the random synthetic weights the decoder amplifies the
# rounding of the tensor-core operands to 1.5e-2 at the output: the CPU oracle with bf16-rounded operands
# (oracle/vae.py emulate_bf16) is 1.51e-2 away from the fp32 oracle, the native decoder about as far,
# and the two are 1.46e-2 apart from each other - rounding noise that de-correlates with the summation order, not a
# systematic difference.  So: an absolute bound against fp32, and the native error may not exceed the error the same
# operand rounding causes on the CPU by more than a quarter.
TOL_VAE = 3e-2


def make_vae(dev, seed=1, max_batch=4):
    from oracle import vae as ovae
    vae = lfm_b200.AutoencoderKL(max_batch=max_batch)
    sd = ovae.synthetic_state_dict(ovae.VAEConfig(), seed)
    vae.load_state_dict(sd, strict=True)
    return vae.to(dev).eval(), sd


@pytest.mark.parametrize("side,B", [(16, 3), (32, 2)])
def test_vae_decode_vs_oracle(dev, side, B):
    """first_stage_model.decode(z).sample (test_flow_latent.py:193) through lfm_create_vae / lfm_decode against the
    fp32 restatement of the diffusers decoder (oracle/vae.py; parity unpinned: diffusers is absent).  side 16 = 128 x 128
    images (whole-row conv tiles up to 128 pixels), side 32 = the 256 x 256 images of every LFM preset (the last stage
    runs on 128-pixel row segments); odd batch, batch larger than one decode chunk."""
    from oracle import vae as ovae
    vae, sd = make_vae(dev, 1, max_batch=2)
    g = torch.Generator().manual_seed(100 + side)
    z = torch.randn(B, 4, side, side, generator=g) / 0.18215 * 0.2       # latents / scale_factor, realistic magnitude
    out = vae.decode(z.to(dev)).sample
    assert out.shape == (B, 3, 8 * side, 8 * side) and torch.isfinite(out).all()
    ref = ovae.vae_decode(sd, z)
    assert rel_l2(out.cpu(), ref) < TOL_VAE
    emu = ovae.vae_decode(sd, z, emulate_bf16=True)                           # what bf16 operands cost in exact fp32 arithmetic
    noise_floor = rel_l2(emu, ref)
    assert rel_l2(out.cpu(), ref) < 1.25 * noise_floor + 1e-3, (rel_l2(out.cpu(), ref), noise_floor)
    assert torch.equal(out, vae.decode(z.to(dev)).sample)                  # deterministic
    assert rel_l2(vae.decode(z[:1].to(dev)).sample.cpu(), out[:1].cpu()) < 1e-5   # samples are independent
    # fused post-processing == the reference's expression applied to the native sample, bit for bit
    u8 = vae.decode_to_uint8(z.to(dev))
    assert u8.dtype == torch.uint8 and u8.shape == (B, 8 * side, 8 * side, 3)
    assert torch.equal(u8.cpu(), ovae.to_uint8_nhwc(out.cpu()))
    # and close to the oracle's image in grey levels: the 1.5e-2 operand-rounding noise on values of magnitude ~0.3 is
    # ~0.6 of a level rms (a few % of the pixels off by more than one level).  Its worst pixels sit in the decoder's high-gain
    # regions, where the CPU emulation of the same operand rounding is itself up to 8 levels off: the native maximum may
    # exceed that floor by one level, and 8 levels otherwise (measured on an H100: native 9 levels where the emulation is 8 at
    # side 32; 4.2 % of the pixels off by more than one level, 0.8 % by more than two)
    d = (u8.cpu().int() - ovae.to_uint8_nhwc(ref).int()).abs()
    d_emu = int((ovae.to_uint8_nhwc(emu).int() - ovae.to_uint8_nhwc(ref).int()).abs().max())
    assert int(d.max()) <= max(8, d_emu + 1) and float((d > 1).float().mean()) < 0.08 and float((d > 2).float().mean()) < 0.01


def test_vae_mid_attention_and_stage_features(dev):
    """Localisation test: the decoder stage by stage is only observable through its output, so perturb-and-compare:
    zeroing the mid-block attention's output projection must change the native result exactly as it changes the
    oracle's (the attention path is live and correct), and a legacy-named checkpoint decodes identically."""
    from oracle import vae as ovae
    vae, sd = make_vae(dev, 2)
    z = torch.randn(1, 4, 16, 16, generator=torch.Generator().manual_seed(5)) * 1.2
    base = vae.decode(z.to(dev)).sample.cpu()
    sd2 = dict(sd)
    sd2["decoder.mid_block.attentions.0.to_out.0.weight"] = torch.zeros_like(sd["decoder.mid_block.attentions.0.to_out.0.weight"])
    sd2["decoder.mid_block.attentions.0.to_out.0.bias"] = torch.zeros_like(sd["decoder.mid_block.attentions.0.to_out.0.bias"])
    vae.load_state_dict(sd2, strict=True)
    noattn = vae.decode(z.to(dev)).sample.cpu()
    d_native, d_ref = base - noattn, ovae.vae_decode(sd, z) - ovae.vae_decode(sd2, z)
    assert float(d_ref.abs().mean()) > 1e-3                                   # the attention matters in the oracle
    assert rel_l2(d_native, d_ref) < 0.1                                      # and changes the native output the same way
    legacy = {k.replace(".to_q.", ".query.").replace(".to_k.", ".key.").replace(".to_v.", ".value.").replace(".to_out.0.", ".proj_attn."): v
              for k, v in sd.items()}
    vae.load_state_dict(legacy, strict=True)
    assert torch.equal(vae.decode(z.to(dev)).sample.cpu(), base)


# ------------------------------------------------------------------------------------------------ edges / CLI


@pytest.mark.parametrize("B", [1, 3, 5])
def test_odd_batch_sizes_and_ctx_growth(dev, B):
    """Ragged sizes: token rows B*256 that are not a multiple of the 256-row pair tile per sample count, the native
    context being re-created when a larger batch arrives, and the uniform-conditioning shortcut vs explicit vectors."""
    g = load_golden("mini_cond")
    cfg = cfg_from_golden(g)
    sd = odit.synthetic_state_dict(cfg, int(g["weight_seed"]))
    net = make_net(cfg, sd, dev)
    gen = torch.Generator().manual_seed(100 + B)
    x = torch.randn(B, 4, 32, 32, generator=gen)
    y = torch.randint(0, cfg.num_classes, (B,), generator=gen)
    t = torch.rand(B, generator=gen)
    v = net(t.to(dev), x.to(dev), y.to(dev))
    assert rel_l2(v.cpu(), odit.dit_forward(sd, cfg, t, x, y)) < TOL_NFE
    # y=None + 0-d t (one shared conditioning row, stride-0 modulation table) == explicit null labels + [B] times
    v0 = net(torch.tensor(0.37, device=dev), x.to(dev))
    v1 = net(torch.full((B,), 0.37, device=dev), x.to(dev), torch.full((B,), cfg.table_rows - 1, device=dev))
    assert rel_l2(v0.cpu(), v1.cpu()) < 1e-6
    # a larger batch afterwards forces a bigger native context; results stay consistent
    xb = torch.cat([x, x, x], 0).to(dev)
    vb = net(torch.tensor(0.37, device=dev), xb)
    assert rel_l2(vb[:B].cpu(), v0.cpu()) < 1e-6 and rel_l2(vb[2 * B:].cpu(), v0.cpu()) < 1e-6


def test_cli_end_to_end(dev, tmp_path):
    """The test_flow_latent.py-compatible CLI (R1/R4): synthetic weights, Karras Heun with CFG, latents saved."""
    import numpy as np
    from lfm_b200 import cli
    out = str(tmp_path)
    rc = cli.main(["--model_type", "DiT-B/2", "--image_size", "256", "--num_in_channels", "4", "--num_classes", "1000",
                   "--label_dropout", "0.1", "--cfg_scale", "1.5", "--batch_size", "4", "--use_karras_samplers",
                   "--method", "heun", "--num_steps", "4", "--synthetic_init", "3", "--n_sample", "16", "--no_decode",
                   "--out_dir", out, "--device", "cuda:0"])
    assert rc == 0
    z = np.load(out + "/samples_cifar10_heun_4_cfg1.5_latents.npy")
    assert z.shape == (4, 4, 32, 32) and np.isfinite(z).all() and np.abs(z).mean() > 0.1
    # torchdiffeq-style entry + NFE counting mode
    rc = cli.main(["--model_type", "DiT-B/2", "--image_size", "256", "--num_in_channels", "4", "--num_classes", "1",
                   "--label_dropout", "0.", "--batch_size", "2", "--method", "euler", "--step_size", "0.25",
                   "--synthetic_init", "3", "--n_sample", "8", "--no_decode", "--out_dir", out, "--device", "cuda:0",
                   "--compute_nfe", "--measure_reps", "2"])
    assert rc == 0


def test_cli_decode_and_generation_loop(dev, tmp_path):
    """The CLI with the native VAE (synthetic decoder weights): default mode writes the image grid from the all-gathered
    uint8 images; --compute_fid runs the generation loop with the fused post-processing and the asynchronous JPEG sink
    (test_flow_latent_ddp.py:116-143: file index j * world + rank + total); --measure_time includes the decode."""
    import os
    from PIL import Image
    from lfm_b200 import cli
    out = str(tmp_path)
    common = ["--model_type", "DiT-B/2", "--image_size", "256", "--num_in_channels", "4", "--num_classes", "1", "--label_dropout", "0.",
              "--method", "euler", "--step_size", "0.25", "--synthetic_init", "3", "--synthetic_vae", "2", "--out_dir", out,
              "--device", "cuda:0", "--dataset", "celeba_256", "--exp", "t"]
    assert cli.main(common + ["--batch_size", "4"]) == 0
    img = Image.open(os.path.join(out, "samples_celeba_256_euler_1e-05_1e-05.jpg"))
    assert img.size == (1024, 256)                                   # 4 images of 256 x 256 in one row (nrow=8)
    assert cli.main(common + ["--batch_size", "3", "--n_sample", "6", "--compute_fid"]) == 0
    d = os.path.join(out, "generated_samples", "celeba_256", "expt_ep1000_meuler_s40")
    files = sorted(os.listdir(d), key=lambda f: int(f.split(".")[0]))
    assert files == [f"{i}.jpg" for i in range(6)]
    assert all(Image.open(os.path.join(d, f)).size == (256, 256) for f in files)
    assert cli.main(common + ["--measure_time", "--measure_reps", "3"]) == 0
    # FID on the device inside the same loop (seeded Inception weights: plumbing, not a meaningful number): statistics
    # file in the reference's pickled-dict layout, the value printed and appended to --output_log (test_flow_latent.py:280-282)
    import numpy as np
    stat, log = os.path.join(out, "stat.npy"), os.path.join(out, "fid.log")
    rng = np.random.RandomState(0)
    feats = rng.rand(64, 2048)
    np.save(stat, {"mu": feats.mean(0), "sigma": np.cov(feats, rowvar=False)}, allow_pickle=True)
    assert cli.main(common + ["--batch_size", "3", "--n_sample", "6", "--compute_fid", "--synthetic_inception", "1", "--no_save",
                              "--real_img_dir", stat, "--output_log", log, "--dataset", "custom"]) == 0
    line = open(log).read().strip()
    assert line.startswith("Epoch = 1000, FID = ") and np.isfinite(float(line.split("FID = ")[1])) and float(line.split("FID = ")[1]) > 0

