"""Semantic synthesis on the GPU: lfm_label_condition against an fp64 histogram reference, SpatialRescaler.forward_labels
against the reference module's fixture (tests/golden/spatial_rescaler.npz) and against the torch one-hot route, the
mask-to-image command line end to end, and the two-path FID command line.

The error bound of one output, out[b, k, i, j] = sum_c w[k, c] n_c / f^2 accumulated with one fmaf per class, is
(K + 2) 2^-24 sum_c |w[k, c]| n_c / f^2 (K roundings of partial sums bounded by that magnitude, plus slack)."""
import ctypes as C
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from lfm_b200 import _lib, cli_semantic, fid
from lfm_b200.downstream import SpatialRescaler

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


def P(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def label_condition(seg, w, stages):
    """lfm_label_condition on a [B, H, W] uint8 map and a [O, K] fp32 weight."""
    B, H, W = seg.shape
    O, K = w.shape
    f = 2 ** stages
    out = torch.full((B, O, H // f, W // f), float("nan"), device=seg.device)
    _lib.check(_lib.load().lfm_label_condition(P(seg), B, H, W, K, stages, P(w), O, P(out), None))
    torch.cuda.synchronize()
    return out


def reference(seg, w, stages):
    """fp64 block histograms n_c / f^2 contracted with w, and the bound above.  Labels >= K are not counted."""
    B, H, W = seg.shape
    O, K = w.shape
    f = 2 ** stages
    oh = F.one_hot(seg.long(), 256)[..., :K].double()                                # [B, H, W, K]
    frac = oh.reshape(B, H // f, f, W // f, f, K).sum((2, 4)) / (f * f)              # [B, Ho, Wo, K]
    ref = torch.einsum("bijc,kc->bkij", frac, w.double())
    mag = torch.einsum("bijc,kc->bkij", frac, w.double().abs())
    return ref, (K + 2) * 2.0 ** -24 * mag


def assert_within(out, ref, bound, what):
    err = (out.double() - ref).abs()
    bad = err > bound
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} outputs outside the bound (max error {float(err.max()):.3g})"


def label_maps(B, H, W, K, stages, seed, dev):
    """Half random labels, half piecewise-constant regions (2^stages-aligned rectangles of one class)."""
    g = torch.Generator().manual_seed(seed)
    f = 2 ** stages
    rnd = torch.randint(0, K, (B, H, W), generator=g)
    coarse = torch.randint(0, K, (B, max(1, H // (4 * f)), max(1, W // (4 * f))), generator=g)
    blocky = F.interpolate(coarse[:, None].float(), size=(H, W), mode="nearest")[:, 0].long()
    seg = torch.where(torch.arange(B)[:, None, None] % 2 == 0, rnd, blocky)
    return seg.to(torch.uint8).to(dev)


# ------------------------------------------------------------------------------------------------ lfm_label_condition


@pytest.mark.parametrize("K", [19, 151, 182, 256])
@pytest.mark.parametrize("stages", [0, 1, 2, 3, 4])
def test_label_condition_vs_fp64(dev, K, stages):
    for H, W in ((256, 256), (512, 256)):
        for O in (4, 16):
            seg = label_maps(2, H, W, K, stages, 1000 * K + 10 * stages + O, dev)
            w = (torch.randn(O, K, generator=torch.Generator().manual_seed(K + O)) / K ** 0.5).to(dev)
            out = label_condition(seg, w, stages)
            ref, bound = reference(seg, w, stages)
            assert_within(out, ref, bound, f"K {K}, stages {stages}, {H}x{W}, out_ch {O}")
            assert torch.equal(out, label_condition(seg, w, stages)), "not bit-identical across calls"


@pytest.mark.parametrize("K,stages", [(19, 3), (256, 4), (182, 0)])
def test_single_class_blocks_are_the_weight_column(dev, K, stages):
    f = 2 ** stages
    g = torch.Generator().manual_seed(K)
    cls = torch.randint(0, K, (2, 256 // f, 256 // f), generator=g)
    seg = cls.repeat_interleave(f, 1).repeat_interleave(f, 2).to(torch.uint8).to(dev)
    w = torch.randn(16, K, generator=g).to(dev)
    out = label_condition(seg, w, stages)
    assert torch.equal(out, w[:, cls.to(dev)].permute(1, 0, 2, 3))


def test_labels_out_of_range_are_not_counted(dev):
    seg = label_maps(2, 256, 256, 19, 3, 5, dev)
    seg[:, ::3, ::5] = 255
    seg[:, 7::11, :] = 19
    w = torch.randn(4, 19, generator=torch.Generator().manual_seed(3)).to(dev)
    out = label_condition(seg, w, 3)
    ref, bound = reference(seg, w, 3)
    assert_within(out, ref, bound, "labels >= K")


# ------------------------------------------------------------------------------------------------ forward_labels


def test_forward_labels_matches_the_reference_fixture(dev):
    z = np.load(os.path.join(GOLDEN, "spatial_rescaler.npz"))
    m = SpatialRescaler(n_stages=3, in_channels=19, out_channels=4, multiplier=0.5)
    m.load_state_dict({"channel_mapper.weight": torch.from_numpy(z["weight"])}, strict=True)
    m = m.to(dev).eval()
    seg = torch.from_numpy(z["seg"]).to(dev)
    out = m.forward_labels(seg)
    assert out.shape == (2, 4, 32, 32) and out.dtype == torch.float32
    ref_out = torch.from_numpy(z["out"]).to(dev)
    _, bound = reference(seg, m.channel_mapper.weight.detach().reshape(4, 19), 3)
    assert_within(out, ref_out.double(), bound, "reference SpatialRescaler")
    assert float((out.double() - ref_out.double()).norm() / ref_out.double().norm()) < 1e-6
    assert torch.equal(m.forward_labels(seg.long()), out)                            # int64 input: the same kernel

    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        with torch.no_grad():
            torch_out = m(F.one_hot(seg.long(), 19).permute(0, 3, 1, 2).float())
    finally:
        torch.backends.cudnn.allow_tf32 = tf32
    assert_within(out, torch_out.double(), bound, "torch forward on the one-hot")


def test_forward_labels_validates_the_labels(dev):
    m = SpatialRescaler(n_stages=3, in_channels=19, out_channels=4).to(dev)
    seg = torch.zeros(1, 64, 64, dtype=torch.uint8, device=dev)
    seg[0, 5, 9] = 19
    with pytest.raises(ValueError, match=r"\[0, 19\)"):
        m.forward_labels(seg)
    neg = torch.zeros(1, 64, 64, dtype=torch.int64, device=dev)
    neg[0, 1, 1] = -1
    with pytest.raises(ValueError, match=r"\[0, 19\)"):
        m.forward_labels(neg)


# ------------------------------------------------------------------------------------------------ command line


def write_masks(root, n, side=512):
    from PIL import Image
    root.mkdir()
    for i in range(n):
        seg = label_maps(1, side, side, 19, 5, 70 + i, "cpu")[0].numpy()
        Image.fromarray(seg).save(root / f"{27000 + i}.png")
    return str(root)


def test_semantic_cli(dev, tmp_path):
    """test_flow_latent_semantic_syn.py with synthetic UNet, rescaler and VAE at the reference's default UNet flags, batch 2
    over five 512-pixel label maps (a partial last batch), Euler at step 0.25: files 0..4, and the first batch equal to the
    same steps composed from the library calls."""
    from PIL import Image
    from lfm_b200.downstream import WrapperCondFlow, sample_from_model
    masks = write_masks(tmp_path / "masks", 5)
    common = ["--dataset", "celeba", "--batch_size", "2", "--synthetic_init", "1", "--synthetic_vae", "2", "--mask_dir", masks,
              "--num_workers", "0", "--device", "cuda:0", "--seed", "7"]
    argv = common + ["--method", "euler", "--step_size", "0.25", "--num_images", "5", "--out_dir", str(tmp_path / "euler")]
    assert cli_semantic.main(argv) == 0
    d = tmp_path / "euler" / "mask2image_generated_samples" / "celeba"
    assert sorted(os.listdir(d)) == [f"{i}.jpg" for i in range(5)]
    assert all(Image.open(d / f).size == (256, 256) for f in os.listdir(d))

    args = cli_semantic.parse_args(argv)
    model, cond, vae = cli_semantic.load(args, dev)
    ds = cli_semantic.CelebAMaskSegmentation(masks, 5)
    seg = torch.stack([ds[0], ds[1]]).to(dev)

    torch.manual_seed(7)
    torch.cuda.manual_seed_all(7)
    u8 = cli_semantic.synthesize(args, model, cond, vae, seg)

    torch.manual_seed(7)
    torch.cuda.manual_seed_all(7)
    c = cond.forward_labels(seg)
    z_0 = torch.randn(2, 4, 32, 32).to(dev)
    fake = sample_from_model(WrapperCondFlow(model, c), z_0, args)[-1]
    x = (vae.decode(fake / args.scale_factor).sample + 1) / 2
    hand = (x * 255 + 0.5).clamp(0, 255).permute(0, 2, 3, 1).to(torch.uint8)
    assert u8.shape == (2, 256, 256, 3)
    assert torch.equal(u8, hand)
    assert float(u8.float().std()) > 1.0

    argv = common + ["--method", "dopri5", "--rtol", "1e-2", "--atol", "1e-2", "--num_images", "2",
                     "--out_dir", str(tmp_path / "dopri5")]
    assert cli_semantic.main(argv) == 0
    assert sorted(os.listdir(tmp_path / "dopri5" / "mask2image_generated_samples" / "celeba")) == ["0.jpg", "1.jpg"]


# ------------------------------------------------------------------------------------------------ FID between two paths


def write_images(root, n, seed):
    from PIL import Image
    root.mkdir()
    g = torch.Generator().manual_seed(seed)
    for i in range(n):
        img = (torch.rand(1, 3, 12, 12, generator=g) * 255)
        img = F.interpolate(img, size=(64, 64), mode="bilinear", align_corners=False)[0].permute(1, 2, 0)
        Image.fromarray(img.round().clamp(0, 255).to(torch.uint8).numpy()).save(root / f"{i:03d}.png")
    return str(root)


def test_fid_cli(dev, tmp_path, capsys):
    a, b = write_images(tmp_path / "a", 7, 1), write_images(tmp_path / "b", 6, 2)
    sd = fid.synthetic_inception_state_dict(1)
    torch.save(sd, tmp_path / "w.pth")
    common = ["--inception_weights", str(tmp_path / "w.pth"), "--batch-size", "4", "--device", "cuda:0"]
    value = fid.main([a, b] + common)
    assert capsys.readouterr().out.startswith("FID:  ")

    from PIL import Image
    net = fid.FIDInception(sd).to(dev)

    def batches(path):
        files = fid.list_images(path)
        for i in range(0, len(files), 4):
            yield torch.from_numpy(np.stack([np.asarray(Image.open(f).convert("RGB")) for f in files[i:i + 4]])).to(dev)

    acc_b = fid.FIDAccumulator(net, dev)
    for x in batches(b):
        acc_b.update(x)
    mu_b, sigma_b = acc_b.stats.finalize()
    np.savez(tmp_path / "b_stats.npz", mu=mu_b.cpu().numpy(), sigma=sigma_b.cpu().numpy())
    acc_a = fid.FIDAccumulator(net, dev)
    for x in batches(a):
        acc_a.update(x)
    want = acc_a.compute(str(tmp_path / "b_stats.npz"))
    assert value > 0 and abs(value - want) <= 1e-9 * abs(want)
    assert abs(fid.main([a, str(tmp_path / "b_stats.npz")] + common) - want) <= 1e-9 * abs(want)

    # A directory against itself: zero up to rounding.  The covariance of 7 images has rank 6, and each of the ~2042 zero
    # eigenvalues of S^1/2 S S^1/2 carries fp64 rounding noise of about 2^-52 lambda_max^2, whose square root (2^-26
    # lambda_max) enters Tr sqrt(...): the floor is 2 D 2^-26 lambda_max (measured on an H100: 5e-2 of it).
    self_value = fid.main([a, a] + common)
    _, sigma_a = acc_a.stats.finalize()
    floor = 2 * 2048 * 2.0 ** -26 * float(torch.linalg.eigvalsh(sigma_a).max())
    assert abs(self_value) < floor < 1e-3 * value
