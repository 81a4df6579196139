"""CPU-side checks of the native VAE encoder and the inpainting command line: the module's key sets and loading, the synthetic
weights, the refusals of encode and of the C entries (all made before the device is touched), the oracle's Downsample2D and
FLOP count, and the command line's dataset reader and flags."""
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import lfm_b200
from lfm_b200 import vae as lvae
from oracle import vae as ovae
from tests.tools import vae_encoder_oracle as oenc


@pytest.fixture(scope="module")
def lib():
    from lfm_b200 import _lib, build
    build.build()
    return _lib.load()


def refused(rc, word):
    from lfm_b200 import _lib
    assert rc != 0
    assert word in _lib.last_error(), _lib.last_error()


def test_key_sets():
    full = lfm_b200.AutoencoderKL(with_encoder=True).state_dict()
    assert len(full) == 248
    shapes = oenc.full_param_shapes()
    assert set(full) == set(shapes)
    assert all(tuple(full[k].shape) == shapes[k] for k in shapes)
    assert len(oenc.encoder_param_shapes()) == 108
    assert len(lfm_b200.AutoencoderKL().state_dict()) == 140
    assert not hasattr(lfm_b200.AutoencoderKL(), "encoder")


def _legacy(sd):
    legacy = {"to_q": "query", "to_k": "key", "to_v": "value", "to_out.0": "proj_attn"}
    out = {}
    for k, v in sd.items():
        for new, old in legacy.items():
            if f"attentions.0.{new}." in k:
                k = k.replace(f"attentions.0.{new}.", f"attentions.0.{old}.")
        out[k] = v
    return out


def test_legacy_full_checkpoint_loads_strictly():
    sd = oenc.synthetic_state_dict(seed=5)
    leg = _legacy(sd)
    assert "encoder.mid_block.attentions.0.query.weight" in leg and "decoder.mid_block.attentions.0.proj_attn.bias" in leg
    vae = lfm_b200.AutoencoderKL(with_encoder=True)
    vae.load_state_dict(leg, strict=True)
    got = vae.state_dict()
    assert all(torch.equal(got[k], sd[k]) for k in sd)
    # the decoder-only module takes the same full checkpoint and ignores the encoder half
    dec = lfm_b200.AutoencoderKL()
    dec.load_state_dict(leg, strict=True)
    # one encoder entry missing: the strict load fails
    leg.pop("encoder.down_blocks.1.resnets.0.conv_shortcut.weight")
    with pytest.raises(RuntimeError, match="conv_shortcut"):
        lfm_b200.AutoencoderKL(with_encoder=True).load_state_dict(leg, strict=True)


def test_from_pretrained_with_encoder(tmp_path):
    import json
    sd = _legacy(oenc.synthetic_state_dict(seed=2))
    (tmp_path / "config.json").write_text(json.dumps({"block_out_channels": [128, 256, 512, 512], "latent_channels": 4}))
    torch.save(sd, tmp_path / "diffusion_pytorch_model.bin")
    assert len(lfm_b200.AutoencoderKL.from_pretrained(str(tmp_path)).state_dict()) == 140
    vae = lfm_b200.AutoencoderKL.from_pretrained(str(tmp_path), with_encoder=True)
    assert len(vae.state_dict()) == 248
    assert torch.equal(vae.state_dict()["encoder.mid_block.attentions.0.to_k.weight"],
                       sd["encoder.mid_block.attentions.0.key.weight"])


def test_synthetic_weights_agree():
    full, dec = lfm_b200.AutoencoderKL(with_encoder=True), lfm_b200.AutoencoderKL()
    a, b = lvae.synthetic_vae_state_dict(full, 3), lvae.synthetic_vae_state_dict(dec, 3)
    assert len(a) == 248 and len(b) == 140
    assert all(torch.equal(a[k], b[k]) for k in b)
    o = oenc.synthetic_state_dict(seed=3)
    assert set(o) == set(a) and all(torch.equal(a[k], o[k]) for k in o)


def test_native_upload_sees_only_its_own_keys():
    vae = lfm_b200.AutoencoderKL(with_encoder=True)
    dec_keys = set(vae._native_state_dict())
    enc_keys = set(vae._enc_native._native_state_dict())
    assert len(dec_keys) == 140 and all(k.startswith(("decoder.", "post_quant_conv.")) for k in dec_keys)
    assert len(enc_keys) == 108 and all(k.startswith(("encoder.", "quant_conv.")) for k in enc_keys)
    # the encoder context shares the module's parameters: no copy
    assert vae._enc_native.encoder.conv_in.weight is vae.encoder.conv_in.weight
    assert enc_keys == set(oenc.encoder_param_shapes())


def test_encode_refusals():
    vae = lfm_b200.AutoencoderKL(with_encoder=True)
    with pytest.raises(RuntimeError, match="CUDA"):
        vae.encode(torch.zeros(1, 3, 128, 128))
    with pytest.raises(RuntimeError, match="with_encoder=True"):
        lfm_b200.AutoencoderKL().encode(torch.zeros(1, 3, 128, 128))


def test_gaussian_distribution():
    mean = torch.randn(2, 4, 3, 3)
    logvar = torch.randn(2, 4, 3, 3)
    d = lvae.DiagonalGaussianDistribution(mean, logvar)
    assert torch.equal(d.mode(), mean)
    assert torch.equal(d.std, torch.exp(0.5 * logvar)) and torch.equal(d.var, torch.exp(logvar))
    g = torch.Generator().manual_seed(7)
    s = d.sample(generator=g)
    eps = torch.randn(mean.shape, generator=torch.Generator().manual_seed(7))
    assert torch.equal(s, mean + torch.exp(0.5 * logvar) * eps)


def test_create_vae_encoder_refusals(lib):
    from lfm_b200 import _lib
    ctx = ctypes.c_void_p()

    def desc(latent, boc=(128, 256, 512, 512), image_ch=3):
        return _lib.VaeDesc(latent, 4, image_ch, len(boc), (ctypes.c_int32 * 8)(*boc), 2, 32)

    refused(lib.lfm_create_vae_encoder(ctypes.byref(desc(8)), 0, ctypes.byref(ctx)), "latent_size")
    refused(lib.lfm_create_vae_encoder(ctypes.byref(desc(128)), 0, ctypes.byref(ctx)), "image side 1024")
    refused(lib.lfm_create_vae_encoder(ctypes.byref(desc(32, image_ch=4)), 0, ctypes.byref(ctx)), "out_channels")
    refused(lib.lfm_create_vae_encoder(ctypes.byref(desc(32, (128, 256, 512, 384))), 0, ctypes.byref(ctx)), "mid-block width")
    refused(lib.lfm_create_vae_encoder(None, 0, ctypes.byref(ctx)), "null")
    rc = lib.lfm_create_vae_encoder(ctypes.byref(desc(32)), 0, ctypes.byref(ctx))
    if torch.cuda.is_available():
        assert rc == 0, _lib.last_error()
        lib.lfm_destroy(ctx)
    else:
        refused(rc, "no CUDA device")
    refused(lib.lfm_encode(None, None, 1, None, None, None), "null ctx")


def test_dbg_conv_down_refusals(lib):
    """lfm_dbg_conv_down(x, w, bias, out, gn_bins, B, side, Cin, Cout, stride, block_n, epi, ksplit, stream)."""
    conv = lib.lfm_dbg_conv_down
    d = ctypes.c_void_p(64)   # never dereferenced: each call is refused on its arguments
    refused(conv(d, d, d, d, None, 1, 256, 128, 128, 1, 0, 3, -1, None), "stride")
    refused(conv(d, d, d, d, None, 1, 384, 128, 128, 2, 0, 3, -1, None), "side")
    refused(conv(d, d, d, d, None, 1, 1024, 128, 128, 2, 0, 3, -1, None), "side")
    refused(conv(d, d, d, d, None, 1, 4, 128, 128, 2, 0, 3, -1, None), "side")
    refused(conv(d, d, d, d, None, 0, 256, 128, 128, 2, 0, 3, -1, None), "B")
    refused(conv(d, d, d, d, None, 1, 256, 96, 128, 2, 0, 3, -1, None), "Cin")
    refused(conv(d, d, d, d, None, 1, 256, 128, 12, 2, 0, 3, -1, None), "Cout")
    refused(conv(d, d, d, d, None, 1, 256, 128, 128, 2, 64, 3, -1, None), "block_n")
    refused(conv(d, d, d, d, None, 1, 256, 128, 128, 2, 0, 1, -1, None), "epi")
    refused(conv(d, d, d, d, None, 1, 256, 128, 128, 2, 0, 3, 9, None), "ksplit")
    refused(conv(None, d, d, d, None, 1, 256, 128, 128, 2, 0, 3, -1, None), "NULL")


def test_dbg_conv_in_takes_512_pixel_images(lib):
    """The encoder's conv_in runs at 512 pixels with 3 channels; other channel counts keep the 256 limit."""
    ci = lib.lfm_dbg_conv_in
    d = ctypes.c_void_p(64)
    refused(ci(d, 4, 4 * 512 * 512, None, 0, 0, d, d, d, 1, 512, 128, None), "side")
    refused(ci(d, 3, 3 * 1024 * 1024, None, 0, 0, d, d, d, 1, 1024, 128, None), "side")
    rc = ci(d, 3, 3 * 512 * 512 - 1, None, 0, 0, d, d, d, 1, 512, 128, None)   # passes the side rule, refused on a_stride
    refused(rc, "a_stride")


def test_oracle_downsample_is_pad_then_stride2():
    g = torch.Generator().manual_seed(0)
    x, w, b = torch.randn(2, 8, 16, 16, generator=g), torch.randn(8, 8, 3, 3, generator=g), torch.randn(8, generator=g)
    ref = F.conv2d(F.pad(x, (0, 1, 0, 1)), w, b, stride=2)
    assert ref.shape == (2, 8, 8, 8)
    assert torch.equal(oenc.downsample(x, w, b), ref)


def test_encode_flops():
    assert round(oenc.encode_flops_per_image(image_side=256) / 1e12, 3) == 0.273
    assert round(oenc.encode_flops_per_image(image_side=512) / 1e12, 3) == 1.117
    vae = lfm_b200.AutoencoderKL(with_encoder=True)
    assert all(vae.encode_flops_per_image(s) == oenc.encode_flops_per_image(image_side=s) for s in (128, 256, 512))


def test_oracle_encode_shapes_and_clamp():
    cfg = ovae.VAEConfig()
    sd = oenc.synthetic_state_dict(cfg, 1)
    sd["quant_conv.bias"] = sd["quant_conv.bias"] + torch.tensor([0, 0, 0, 0, 100.0, -100.0, 0, 0])
    x = torch.rand(1, 3, 128, 128) * 2 - 1
    mean, logvar = oenc.vae_encode(sd, x, cfg)
    assert mean.shape == logvar.shape == (1, 4, 16, 16)
    assert float(logvar[:, 0].min()) == 20.0 and float(logvar[:, 1].max()) == -30.0
    mean_e, _ = oenc.vae_encode(sd, x, cfg, emulate_bf16=True)
    assert not ovae._EMULATE_BF16
    rel = float((mean_e - mean).norm() / mean.norm())
    assert 0 < rel < 0.05


# ------------------------------------------------------------------------------------------------ command line

def _write_pairs(root, n, side=32):
    from PIL import Image
    gt, masks = root / "gt", root / "masks"
    gt.mkdir()
    masks.mkdir()
    rng = np.random.default_rng(0)
    for i in range(n):
        Image.fromarray(rng.integers(0, 256, (side, side, 3), dtype=np.uint8)).save(gt / f"{i:06d}.jpg")
        m = np.full((side, side), 255, np.uint8)
        m[8:20, 4:24] = 0
        m[0, 0] = 77
        Image.fromarray(m).save(masks / f"{i:06d}.png")
    return str(gt), str(masks)


def test_dataset_reader(tmp_path):
    from PIL import Image
    from lfm_b200.cli_inpaint import InpaintingEvalDataset
    gt, masks = _write_pairs(tmp_path, 3)
    ds = InpaintingEvalDataset(gt, masks, 3)
    assert len(ds) == 3
    img, mask, masked = ds[1]
    raw = torch.from_numpy(np.array(Image.open(os.path.join(gt, "000001.jpg")).convert("RGB"))).permute(2, 0, 1).float() / 255.0
    png = torch.from_numpy(np.array(Image.open(os.path.join(masks, "000001.png"))))
    m = 1 - png / 255.0
    assert mask.shape == (1, 32, 32) and img.shape == masked.shape == (3, 32, 32)
    assert torch.equal(img, raw * 2.0 - 1.0)
    assert torch.equal(mask, (m * 2.0 - 1.0).unsqueeze(0))
    assert torch.equal(masked, (1 - m) * raw * 2.0 - 1.0)
    assert float(mask[0, 10, 10]) == 1.0 and float(mask[0, 30, 30]) == -1.0     # 1 marks the hole
    assert float(masked[0, 10, 10]) == -1.0


# (flag, default) of every argument of the reference's parser, downstream_tasks/test_flow_latent_inpainting.py:170-224
REFERENCE_FLAGS = [
    ("seed", 1024), ("compute_fid", False), ("epoch_id", 500), ("image_size", 256), ("num_in_channels", 9),
    ("num_out_channels", 4), ("nf", 256), ("centered", True), ("resamp_with_conv", True), ("num_res_blocks", 2),
    ("num_heads", 4), ("num_head_upsample", -1), ("num_head_channels", -1), ("attn_resolutions", (16, 8)),
    ("ch_mult", (1, 2, 3, 4)), ("dropout", 0.0), ("num_classes", None), ("use_scale_shift_norm", True),
    ("resblock_updown", False), ("use_new_attention_order", False), ("scale_factor", 0.18215), ("exp", "latent_kl_exp1"),
    ("real_img_dir", "./pytorch_fid/cifar10_train_stat.npy"), ("dataset", "celeba_256"), ("num_timesteps", 200),
    ("batch_size", 50), ("atol", 1e-5), ("rtol", 1e-5), ("method", "dopri5"), ("step_size", 0.01), ("perturb", False),
    ("pretrained_autoencoder_ckpt", "../stabilityai/sd-vae-ft-mse"),
]


def test_parser_defaults_are_the_reference_ones():
    from lfm_b200.cli_inpaint import build_parser
    args = build_parser().parse_args([])
    for flag, default in REFERENCE_FLAGS:
        v = getattr(args, flag)
        assert (tuple(v) if isinstance(v, list) else v) == default, flag
    assert (args.gt_dir, args.mask_dir, args.num_images, args.out_dir) == (
        "./gt_celeb/", "./dataset/masks_val_256_small_eval", 2993, ".")


def test_parser_accepts_every_flag():
    from lfm_b200.cli_inpaint import build_parser
    argv = ["--seed", "3", "--compute_fid", "--epoch_id", "7", "--image_size", "128", "--num_in_channels", "9",
            "--num_out_channels", "4", "--nf", "128", "--centered", "--resamp_with_conv", "1", "--num_res_blocks", "1",
            "--num_heads", "2", "--num_head_upsample", "-1", "--num_head_channels", "64", "--attn_resolutions", "8", "4",
            "--ch_mult", "1", "2", "--dropout", "0.0", "--num_classes", "1", "--use_scale_shift_norm", "1", "--resblock_updown", "",
            "--use_new_attention_order", "", "--scale_factor", "0.2", "--exp", "e", "--real_img_dir", "r", "--dataset", "d",
            "--num_timesteps", "10", "--batch_size", "2", "--atol", "1e-4", "--rtol", "1e-4", "--method", "euler",
            "--step_size", "0.25", "--perturb", "--pretrained_autoencoder_ckpt", "p", "--gt_dir", "g", "--mask_dir", "m",
            "--num_images", "2", "--num_workers", "0", "--out_dir", "o", "--device", "cuda:0", "--synthetic_init", "1",
            "--synthetic_vae", "2"]
    a = build_parser().parse_args(argv)
    assert a.attn_resolutions == [8, 4] and a.method == "euler" and a.num_images == 2 and a.synthetic_vae == 2
    assert a.centered is False and a.resblock_updown is False


def test_cli_refuses_without_a_vae(tmp_path):
    from lfm_b200 import cli_inpaint
    args = cli_inpaint.build_parser().parse_args(["--pretrained_autoencoder_ckpt", str(tmp_path / "missing")])
    with pytest.raises(SystemExit, match="encoder"):
        cli_inpaint.load(args, torch.device("cpu"))
