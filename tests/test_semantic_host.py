"""CPU-side checks of semantic synthesis: the command line's flags, dataset refusal, label-map reader and checkpoint loading,
SpatialRescaler.forward_labels' refusals and lfm_label_condition's argument checks (made before the device is touched), and the
two-path FID entry on statistics files and its directory listing."""
import os

import numpy as np
import pytest
import torch

from lfm_b200 import cli_semantic, fid
from lfm_b200.downstream import SpatialRescaler

GOLD_FID = os.path.join(os.path.dirname(__file__), "golden", "fid_ref.npz")

# (flag, default) of every argument of the reference's parser, downstream_tasks/test_flow_latent_semantic_syn.py:154-229
REFERENCE_FLAGS = [
    ("seed", 1024), ("compute_fid", False), ("epoch_id", 425), ("image_size", 256), ("num_in_channels", 8),
    ("num_out_channels", 4), ("nf", 256), ("centered", True), ("resamp_with_conv", True), ("num_res_blocks", 2),
    ("num_heads", 4), ("num_head_upsample", -1), ("num_head_channels", -1), ("attn_resolutions", (8, 4)),
    ("ch_mult", (1, 2, 3, 4)), ("dropout", 0.0), ("num_classes", None), ("use_scale_shift_norm", True),
    ("resblock_updown", False), ("use_new_attention_order", False), ("scale_factor", 0.18215),
    ("exp", "experiment_cifar_default"), ("real_img_dir", "./pytorch_fid/cifar10_train_stat.npy"), ("dataset", "cifar10"),
    ("num_timesteps", 200), ("batch_size", 200), ("atol", 1e-5), ("rtol", 1e-5), ("method", "dopri5"), ("step_size", 0.01),
    ("perturb", False), ("pretrained_autoencoder_ckpt", "../stabilityai/sd-vae-ft-mse"),
]


# ------------------------------------------------------------------------------------------------ flags


def test_parser_defaults_are_the_reference_ones():
    args = cli_semantic.build_parser().parse_args([])
    for flag, default in REFERENCE_FLAGS:
        v = getattr(args, flag)
        assert (tuple(v) if isinstance(v, list) else v) == default, flag
    assert (args.mask_dir, args.num_images, args.num_workers, args.out_dir, args.device) == (
        "dataset/CelebAMask-HQ/mask", 3000, 4, ".", None)
    assert args.synthetic_init is None and args.synthetic_vae is None
    with pytest.raises(SystemExit):
        cli_semantic.build_parser().parse_args(["--method", "heun"])


def test_readme_abbreviation_parses():
    args = cli_semantic.parse_args(["--dataset", "celeba", "--attn_resolution", "16", "8"])
    assert args.attn_resolutions == [16, 8]


@pytest.mark.parametrize("dataset", ["cifar10", "celeba_256", "ade20k", "coco"])
def test_other_datasets_exit_naming_celeba(dataset, capsys):
    argv = [] if dataset == "cifar10" else ["--dataset", dataset]
    with pytest.raises(SystemExit):
        cli_semantic.main(argv)
    err = capsys.readouterr().err
    assert "'celeba'" in err and "supported dataset" in err and dataset in err


# ------------------------------------------------------------------------------------------------ reader


def _write_masks(root, maps):
    from PIL import Image
    root.mkdir(exist_ok=True)
    for i, m in enumerate(maps):
        Image.fromarray(m).save(root / f"{27000 + i}.png")
    return str(root)


def test_reader_indices_start_at_27000(tmp_path):
    maps = [np.full((256, 256), i, np.uint8) for i in range(3)]
    ds = cli_semantic.CelebAMaskSegmentation(_write_masks(tmp_path / "m", maps), 3)
    assert len(ds) == 3
    assert ds.path(0).endswith("27000.png") and ds.path(2).endswith("27002.png")
    for i in range(3):
        seg = ds[i]
        assert seg.dtype == torch.uint8 and seg.shape == (256, 256)
        assert torch.equal(seg, torch.full((256, 256), i, dtype=torch.uint8))


@pytest.mark.parametrize("side", [512, 500, 256, 200])
def test_reader_nearest_resize(tmp_path, side):
    rng = np.random.default_rng(side)
    m = rng.integers(0, 19, (side, side)).astype(np.uint8)
    seg = cli_semantic.CelebAMaskSegmentation(_write_masks(tmp_path / "m", [m]), 1)[0].numpy()
    idx = np.floor(np.arange(256) * (side / 256)).astype(np.int64)
    assert np.array_equal(seg, m[np.ix_(idx, idx)])
    if side == 256:
        assert np.array_equal(seg, m)


@pytest.mark.parametrize("side", [512, 500])
def test_reader_resize_equals_cv2_nearest(tmp_path, side):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(side + 1)
    m = rng.integers(0, 19, (side, side)).astype(np.uint8)
    seg = cli_semantic.CelebAMaskSegmentation(_write_masks(tmp_path / "m", [m]), 1)[0].numpy()
    assert np.array_equal(seg, cv2.resize(m, (256, 256), interpolation=cv2.INTER_NEAREST))


@pytest.mark.parametrize("bad", ["rgb", "non_square", "out_of_range"])
def test_reader_refuses_with_the_file_name(tmp_path, bad):
    m = {"rgb": np.zeros((256, 256, 3), np.uint8), "non_square": np.zeros((256, 240), np.uint8),
         "out_of_range": np.full((256, 256), 19, np.uint8)}[bad]
    ds = cli_semantic.CelebAMaskSegmentation(_write_masks(tmp_path / "m", [m]), 1)
    with pytest.raises(ValueError, match="27000.png"):
        ds[0]


# ------------------------------------------------------------------------------------------------ checkpoints

TINY = ["--dataset", "celeba", "--nf", "64", "--ch_mult", "1", "2", "--num_res_blocks", "1", "--attn_resolutions", "2",
        "--image_size", "32", "--exp", "tiny", "--epoch_id", "3", "--synthetic_vae", "4"]


def test_checkpoints_load_strictly_with_the_module_prefix(tmp_path, monkeypatch):
    ref_model, ref_cond, _ = cli_semantic.load(cli_semantic.parse_args(TINY + ["--synthetic_init", "5"]), torch.device("cpu"))
    d = tmp_path / "saved_info" / "latent_flow_mask2image" / "celeba" / "tiny"
    d.mkdir(parents=True)
    torch.save({"module." + k: v.clone() + 1 for k, v in ref_model.state_dict().items()}, d / "model_3.pth")
    torch.save({"module.channel_mapper.weight": ref_cond.channel_mapper.weight.detach().clone() + 1}, d / "cond_stage_model_3.pth")
    monkeypatch.chdir(tmp_path)
    model, cond, vae = cli_semantic.load(cli_semantic.parse_args(TINY), torch.device("cpu"))
    assert vae is not None and not vae.with_encoder
    assert set(model.state_dict()) == set(ref_model.state_dict())
    for k, v in model.state_dict().items():
        assert torch.equal(v, ref_model.state_dict()[k] + 1), k
    assert list(cond.state_dict()) == ["channel_mapper.weight"]
    assert torch.equal(cond.channel_mapper.weight, ref_cond.channel_mapper.weight + 1)

    torch.save({"module.channel_mapper.weight": ref_cond.channel_mapper.weight.detach(),
                "module.channel_mapper.bias": torch.zeros(4)}, d / "cond_stage_model_3.pth")
    with pytest.raises(RuntimeError, match="Unexpected key"):
        cli_semantic.load(cli_semantic.parse_args(TINY), torch.device("cpu"))
    torch.save({"module.channel_mapper.weight": ref_cond.channel_mapper.weight.detach()}, d / "cond_stage_model_3.pth")
    sd = {"module." + k: v for k, v in ref_model.state_dict().items()}
    sd.pop(next(iter(sd)))
    torch.save(sd, d / "model_3.pth")
    with pytest.raises(RuntimeError, match="Missing key"):
        cli_semantic.load(cli_semantic.parse_args(TINY), torch.device("cpu"))


def test_synthetic_channel_mapper_weight():
    _, cond, _ = cli_semantic.load(cli_semantic.parse_args(TINY + ["--synthetic_init", "5"]), torch.device("cpu"))
    want = torch.randn(4, 19, 1, 1, generator=torch.Generator().manual_seed(5)) / 19 ** 0.5
    assert torch.equal(cond.channel_mapper.weight, want)


def test_cli_refuses_without_a_vae(tmp_path):
    args = cli_semantic.parse_args(["--dataset", "celeba", "--pretrained_autoencoder_ckpt", str(tmp_path / "missing")])
    with pytest.raises(SystemExit, match="synthetic_vae"):
        cli_semantic.load(args, torch.device("cpu"))


# ------------------------------------------------------------------------------------------------ forward_labels refusals


def test_forward_labels_refusals():
    seg = torch.zeros(1, 16, 16, dtype=torch.uint8)
    with pytest.raises(ValueError, match="CUDA"):
        SpatialRescaler(n_stages=3, in_channels=19, out_channels=4).forward_labels(seg)
    with pytest.raises(NotImplementedError, match="bias"):
        SpatialRescaler(n_stages=3, in_channels=19, out_channels=4, bias=True).forward_labels(seg)
    with pytest.raises(NotImplementedError, match="bilinear"):
        SpatialRescaler(n_stages=3, method="nearest", in_channels=19, out_channels=4).forward_labels(seg)
    with pytest.raises(NotImplementedError, match="bilinear"):
        SpatialRescaler(n_stages=3, multiplier=0.25, in_channels=19, out_channels=4).forward_labels(seg)
    with pytest.raises(NotImplementedError, match="out_channels"):
        SpatialRescaler(n_stages=3, in_channels=19).forward_labels(seg)
    with pytest.raises(ValueError, match="uint8 or int64"):
        SpatialRescaler(n_stages=3, in_channels=19, out_channels=4).forward_labels(seg.int())
    with pytest.raises(ValueError, match="multiples"):
        SpatialRescaler(n_stages=3, in_channels=19, out_channels=4).forward_labels(torch.zeros(1, 16, 12, dtype=torch.uint8))


def test_label_condition_entry_refuses_before_touching_the_device():
    import ctypes
    from lfm_b200 import _lib, build
    build.build()
    lib = _lib.load()
    p = ctypes.c_void_p(16)

    def refused(word, *args):
        assert lib.lfm_label_condition(*args) != 0
        assert word in _lib.last_error(), _lib.last_error()

    refused("num_classes", p, 1, 64, 64, 0, 3, p, 4, p, None)
    refused("num_classes", p, 1, 64, 64, 257, 3, p, 4, p, None)
    refused("out_ch", p, 1, 64, 64, 19, 3, p, 0, p, None)
    refused("out_ch", p, 1, 64, 64, 19, 3, p, 17, p, None)
    refused("n_stages", p, 1, 64, 64, 19, -1, p, 4, p, None)
    refused("n_stages", p, 1, 64, 64, 19, 5, p, 4, p, None)
    refused("multiples", p, 1, 60, 64, 19, 3, p, 4, p, None)
    refused("multiples", p, 0, 64, 64, 19, 3, p, 4, p, None)
    refused("NULL", None, 1, 64, 64, 19, 3, p, 4, p, None)


# ------------------------------------------------------------------------------------------------ FID between two paths


def test_fid_of_two_statistics_files(tmp_path, capsys):
    z = np.load(GOLD_FID)
    a, b = str(tmp_path / "a.npz"), str(tmp_path / "b.npy")
    np.savez(a, mu=z["mu1"], sigma=z["s1"])
    np.save(b, {"mu": z["mu2"], "sigma": z["s2"]}, allow_pickle=True)
    torch.save(fid.synthetic_inception_state_dict(1), tmp_path / "w.pth")
    value = fid.main([a, b, "--inception_weights", str(tmp_path / "w.pth"), "--device", "cpu"])
    assert abs(value - float(z["fid"])) < 1e-9 * float(z["fid"])
    out = capsys.readouterr().out
    assert out.startswith("FID:  ") and abs(float(out.split()[-1]) - float(z["fid"])) < 1e-9 * float(z["fid"])


def test_fid_arguments(tmp_path):
    with pytest.raises(SystemExit):
        fid.build_parser().parse_args(["a", "b"])                                      # --inception_weights is required
    with pytest.raises(SystemExit):
        fid.build_parser().parse_args(["a", "b", "--inception_weights", "w", "--dims", "768"])
    a = fid.build_parser().parse_args(["a", "b", "--inception_weights", "w"])
    assert (a.path, a.batch_size, a.device, a.dims) == (["a", "b"], 50, None, 2048)
    with pytest.raises(RuntimeError, match="Invalid path"):
        fid.main([str(tmp_path / "missing"), str(tmp_path), "--inception_weights", "w"])


def test_fid_directory_listing(tmp_path):
    from PIL import Image
    img = Image.fromarray(np.zeros((8, 8, 3), np.uint8))
    for name in ["b.png", "a.jpg", "c.jpeg", "d.webp", "e.bmp", "notes.txt", "f.JPG", "g.npy"]:
        if name.endswith((".txt", ".npy")):
            (tmp_path / name).write_bytes(b"x")
        else:
            img.save(tmp_path / name, format={"jpg": "JPEG", "JPG": "JPEG", "jpeg": "JPEG", "png": "PNG", "webp": "WEBP",
                                              "bmp": "BMP"}[name.rsplit(".", 1)[1]])
    (tmp_path / "sub").mkdir()
    img.save(tmp_path / "sub" / "0.png")
    assert [f.name for f in fid.list_images(str(tmp_path))] == ["a.jpg", "b.png", "c.jpeg", "d.webp", "e.bmp"]


def test_fid_refuses_a_batch_of_mixed_sizes(tmp_path):
    from PIL import Image
    Image.fromarray(np.zeros((8, 8, 3), np.uint8)).save(tmp_path / "0.png")
    Image.fromarray(np.zeros((8, 10, 3), np.uint8)).save(tmp_path / "1.png")
    net = fid.FIDInception(fid.synthetic_inception_state_dict(1))
    with pytest.raises(ValueError, match="differ in size"):
        fid.statistics_of_path(str(tmp_path), net, batch_size=2, device=torch.device("cpu"))
