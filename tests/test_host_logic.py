"""Host-side logic of the drop-in boundary (no GPU): state-dict surface, time grids, RNG-free helpers,
the world_size-2 gather layout on gloo, and that the product refuses to run on CPU."""
import os
import types

import pytest
import torch
import torch.multiprocessing as mp

import lfm_b200
from lfm_b200 import dist as ldist
from lfm_b200.synthetic import synthetic_state_dict
from oracle import dit as odit
from oracle import solvers as osol


def _mini(**kw):
    args = dict(img_resolution=32, patch_size=2, in_channels=4, hidden_size=256, depth=2, num_heads=4, label_dropout=0.1,
                num_classes=10)
    args.update(kw)
    return lfm_b200.DiT(**args)


def test_state_dict_surface_matches_reference_keys():
    # oracle.param_shapes is pinned to the reference by oracle/make_goldens.py (load_state_dict strict=True)
    net = _mini()
    cfg = odit.DiTConfig(hidden_size=256, depth=2, num_heads=4, label_dropout=0.1, num_classes=10)
    want = odit.param_shapes(cfg)
    got = {k: tuple(v.shape) for k, v in net.state_dict().items()}
    assert got == want
    assert list(got) == list(want)  # same registration order
    with torch.device("meta"):
        big = lfm_b200.DiT_models["DiT-L/2"](img_resolution=32, in_channels=4, label_dropout=0.0, num_classes=1)
    assert len(big.state_dict()) == 252


def test_every_dit_models_entry_has_the_reference_key_table():
    """All twelve entries of models/DiT.py:355-415 (patch 2 / 4 / 8, head_dim 64 and 72) at latent sides 32 and 64: same keys, shapes and order
    as the oracle's table, which the reference modules pin for these geometries too (tests/golden/mini_p4 ... mini_r64p2)."""
    for name, kw in odit.DIT_PRESETS.items():
        for side in (32, 64):
            with torch.device("meta"):
                net = lfm_b200.DiT_models[name](img_resolution=side, in_channels=4, label_dropout=0.1, num_classes=1000)
            cfg = odit.make_config(name, img_resolution=side, label_dropout=0.1, num_classes=1000)
            want = odit.param_shapes(cfg)
            got = {k: tuple(v.shape) for k, v in net.state_dict().items()}
            assert got == want and list(got) == list(want), (name, side)


def test_padded_head_major_attention_layout_is_equivalent():
    """The layout contract of the mma.sync attention kernels (csrc/kernels.cuh qkv_src_row / dit_proj_weight_pad_kernel,
    restated here): qkv rows re-ordered head-major with head_dim 72 zero-padded to 80, proj columns padded to match.  Attention computed
    in that layout (scale 72^-1/2) followed by the padded projection equals timm's Attention on the original weights."""
    D, H, dh, dhp, T, B = 1152, 16, 72, 80, 16, 2
    g = torch.Generator().manual_seed(5)
    wq, bq = torch.randn(3 * D, D, generator=g) * 0.03, torch.randn(3 * D, generator=g) * 0.1
    wp, bp = torch.randn(D, D, generator=g) * 0.03, torch.randn(D, generator=g) * 0.1
    x = torch.randn(B, T, D, generator=g)
    cfg = odit.DiTConfig(hidden_size=D, depth=1, num_heads=H)
    want = odit.attention({"a.qkv.weight": wq, "a.qkv.bias": bq, "a.proj.weight": wp, "a.proj.bias": bp}, "a.", cfg, x)
    # destination row r = head * 3 dhp + which * dhp + d  <-  source row which * D + head * dh + d  (zero for d >= dh)
    r = torch.arange(3 * H * dhp)
    h, which, d = r // (3 * dhp), (r % (3 * dhp)) // dhp, r % dhp
    src = (which * D + h * dh + d).clamp(max=3 * D - 1)
    live = (d < dh)
    wq2 = torch.where(live[:, None], wq[src], torch.zeros(()))
    bq2 = torch.where(live, bq[src], torch.zeros(()))
    # destination column c = head * dhp + d  <-  source column head * dh + d
    c = torch.arange(H * dhp)
    hc, dc = c // dhp, c % dhp
    wp2 = torch.where((dc < dh)[None, :], wp[:, (hc * dh + dc).clamp(max=D - 1)], torch.zeros(()))
    qkv = (x @ wq2.T + bq2).reshape(B, T, H, 3, dhp).permute(3, 0, 2, 1, 4)     # [3, B, H, T, dhp]
    o = torch.softmax((qkv[0] @ qkv[1].transpose(-1, -2)) * dh ** -0.5, dim=-1) @ qkv[2]
    assert float(o[..., dh:].abs().max()) == 0.0                                 # padded output channels are exactly zero
    got = o.transpose(1, 2).reshape(B, T, H * dhp) @ wp2.T + bp
    assert float((got - want).norm() / want.norm()) < 1e-5


def test_reference_init_is_degenerate_and_synthetic_is_not():
    net = _mini()
    assert float(net.final_layer.linear.weight.abs().max()) == 0.0          # models/DiT.py:225-228
    assert float(net.blocks[0].adaLN_modulation[1].weight.abs().max()) == 0.0
    sd = synthetic_state_dict(net, 5)
    ref = odit.synthetic_state_dict(odit.DiTConfig(hidden_size=256, depth=2, num_heads=4, label_dropout=0.1,
                                                   num_classes=10), 5)
    assert all(torch.equal(sd[k], ref[k]) for k in ref)
    net.load_state_dict(sd, strict=True)
    with pytest.raises(RuntimeError):
        bad = dict(sd)
        bad.pop("pos_embed")
        net.load_state_dict(bad, strict=True)


def test_checkpoint_prefix_strip_roundtrip():
    # test_flow_latent.py:140-141 strips the 7-char "module." prefix before load_state_dict(strict=True)
    net = _mini()
    sd = synthetic_state_dict(net, 2)
    ckpt = {"module." + k: v for k, v in sd.items()}
    for key in list(ckpt.keys()):
        ckpt[key[7:]] = ckpt.pop(key)
    net.load_state_dict(ckpt, strict=True)


def test_euler_time_grid_matches_oracle_restatement():
    for h in (0.5, 0.1, 0.05, 0.02, 0.01, 1 / 3, 0.3):
        a, b = lfm_b200.euler_time_grid(h), osol.tdq_euler_grid(h)
        assert torch.equal(a, b)
    assert len(lfm_b200.euler_time_grid(0.02)) == 51


def test_no_cpu_path():
    net = _mini()
    x = torch.randn(2, 4, 32, 32)
    with pytest.raises(RuntimeError):
        net(torch.tensor(0.5), x)
    with pytest.raises(RuntimeError):
        lfm_b200.karras_sample(net, x, 4, clip_denoised=False, sampler="euler", sigma_min=1e-5, sigma_max=1.0)
    with pytest.raises(NotImplementedError):
        lfm_b200.karras_sample(net, x, 4, clip_denoised=True, sampler="euler")
    with pytest.raises(NotImplementedError):
        lfm_b200.create_network(types.SimpleNamespace(use_origin_adm=False, model_type="ddpm++"))   # SongUNet


def test_create_network_factory():
    cfg = types.SimpleNamespace(use_origin_adm=False, model_type="DiT-B/2", image_size=256, f=8, num_in_channels=4,
                                label_dropout=0.1, num_classes=1000)
    with torch.device("meta"):
        net = lfm_b200.create_network(cfg)
    assert net.hidden_size == 768 and net.depth == 12 and net.table_rows == 1001 and net.img_resolution == 32
    # --model_type DiT-XL/2 --image_size 512: head_dim 72 on 64 x 64 latents (1024 tokens) - models/__init__.py:6-17 maps it the same way
    cfg = types.SimpleNamespace(use_origin_adm=False, model_type="DiT-XL/2", image_size=512, f=8, num_in_channels=4,
                                label_dropout=0.0, num_classes=1)
    with torch.device("meta"):
        net = lfm_b200.create_network(cfg)
    assert (net.hidden_size, net.depth, net.num_heads, net.patch_size, net.img_resolution, net.table_rows) == (1152, 28, 16, 2, 64, 1)
    assert tuple(net.pos_embed.shape) == (1, 1024, 1152)


def test_ddp_index_helpers():
    assert ldist.total_samples(50000, 64, 8) == 50176       # test_flow_latent_ddp.py:116-123
    assert ldist.file_index(3, 8, 5, 512) == 3 * 8 + 5 + 512  # :138
    assert ldist.rank_seed(42, 3) == 45


def _gather_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    import torch.distributed as dist
    r, w, _ = ldist.init_from_env("gloo")
    x = torch.arange(3 * 2, dtype=torch.float32).reshape(3, 2) + 100 * r   # 3 "images" per rank
    out = ldist.all_gather_batch(x)
    q.put((r, out.tolist()))
    dist.barrier()
    dist.destroy_process_group()


def test_all_gather_layout_world2_gloo():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29650 + (os.getpid() % 200)
    procs = [ctx.Process(target=_gather_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=120) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    # image j of rank r lands at j * world + r (the reference's file index, test_flow_latent_ddp.py:138)
    want = [[0, 1], [100, 101], [2, 3], [102, 103], [4, 5], [104, 105]]
    assert res[0] == want and res[1] == want


def test_unet_state_dict_surface_and_factory():
    from oracle import unet as ounet
    cfg = types.SimpleNamespace(use_origin_adm=True, layout=False, image_size=512, num_in_channels=4, nf=256, num_out_channels=4,
                                num_res_blocks=2, attn_resolutions=(16, 8), dropout=0.0, ch_mult=(1, 2, 2, 2, 4),
                                resamp_with_conv=True, num_classes=None, num_heads=4, num_head_channels=-1,
                                num_head_upsample=-1, use_scale_shift_norm=True, resblock_updown=False,
                                use_new_attention_order=False)
    with torch.device("meta"):
        net = lfm_b200.create_network(cfg)            # models/__init__.py:7-8 -> get_flow_model
    want = ounet.param_shapes(ounet.UNetConfig())     # pinned to the reference by oracle/make_goldens.py
    got = {k: tuple(v.shape) for k, v in net.state_dict().items()}
    assert got == want and list(got) == list(want) and len(got) == 396
    cfg.resblock_updown = True
    with pytest.raises(NotImplementedError):
        lfm_b200.create_network(cfg)
    cfg.resblock_updown, cfg.layout = False, True
    with pytest.raises(NotImplementedError):
        lfm_b200.create_network(cfg)
    # zero_module layers start at zero as in the reference (unet.py:198,276,594)
    small = lfm_b200.UNetModel(image_size=32, in_channels=4, model_channels=128, out_channels=4, num_res_blocks=1,
                               attention_resolutions=(2,), channel_mult=(1, 2), num_heads=2, use_scale_shift_norm=True)
    assert float(small.out[2].weight.abs().max()) == 0.0
    from lfm_b200.synthetic import synthetic_unet_state_dict
    sd = synthetic_unet_state_dict(small, 21)
    ref = ounet.synthetic_state_dict(ounet.UNetConfig(image_size=32, model_channels=128, num_res_blocks=1,
                                                      attention_resolutions=(2,), channel_mult=(1, 2), num_heads=2), 21)
    assert all(torch.equal(sd[k], ref[k]) for k in ref)


def test_edm_state_dict_surface_and_factory():
    """create_network -> get_edm_network -> DhariwalUNet (models/__init__.py:10-11, EDM.py:906-921): key set, order and
    shapes of the ffhq_adm / imnet_adm presets, incl. the constant resample_filter buffers; init and error behaviour."""
    from oracle import edm as oedm
    cfg = types.SimpleNamespace(use_origin_adm=False, model_type="adm", image_size=256, f=8, num_in_channels=4,
                                num_out_channels=4, label_dim=1000, nf=256, ch_mult=(1, 2, 3, 4), num_res_blocks=2,
                                attn_resolutions=(16, 8, 4), dropout=0.1, label_dropout=0.1)
    with torch.device("meta"):
        net = lfm_b200.create_network(cfg)
    want = oedm.param_shapes(oedm.EDMConfig(label_dim=1000))      # pinned to the reference by oracle/make_goldens.py
    got = {k: tuple(v.shape) for k, v in net.state_dict().items()}
    assert got == want and list(got) == list(want) and len(got) == 429
    assert sum(k.endswith("resample_filter") for k in got) == 12   # 3 down + 3 up blocks, conv0 + skip each
    cfg.model_type = "adm_context"
    with pytest.raises(NotImplementedError):
        lfm_b200.create_network(cfg)
    small = lfm_b200.DhariwalUNet(img_resolution=16, in_channels=4, out_channels=4, label_dim=5, model_channels=128,
                                  channel_mult=(1, 2), num_blocks=1, attn_resolutions=(8,))
    # init_zero layers start at zero, resample filters at 0.25 (EDM.py:742,96-98)
    assert float(small.out_conv.weight.abs().max()) == 0.0 and float(small.dec["8x8_in0"].proj.weight.abs().max()) == 0.0
    assert torch.all(small.enc["8x8_down"].skip.resample_filter == 0.25)
    from lfm_b200.synthetic import synthetic_edm_state_dict
    sd = synthetic_edm_state_dict(small, 31)
    ref = oedm.synthetic_state_dict(oedm.EDMConfig(img_resolution=16, label_dim=5, model_channels=128, channel_mult=(1, 2),
                                                   num_blocks=1, attn_resolutions=(8,)), 31)
    assert list(sd) == list(ref) and all(torch.equal(sd[k], ref[k]) for k in ref)
    small.load_state_dict(sd, strict=True)
    with pytest.raises(RuntimeError):                              # no CPU path
        small(torch.tensor(0.5), torch.randn(2, 4, 16, 16))
    with pytest.raises(RuntimeError):                              # one_hot semantics: class ids only
        small(torch.tensor(0.5), torch.randn(2, 4, 16, 16), torch.tensor([0, 5]))


def test_sampler_label_validation():
    """The solver entry points validate labels before handing raw pointers to the C ABI (the device kernels clamp):
    one label per network row, each a valid table row - as nn.Embedding / F.one_hot raise in the reference."""
    from lfm_b200 import solvers
    net = _mini(label_dropout=0.0)                       # 10 classes, no null row: y_null = num_classes is out of range
    assert net.table_rows == 10
    ok = solvers._check_labels(net, torch.tensor([0, 9, 3, 3]), 4, "cpu")
    assert ok.dtype == torch.int64 and ok.tolist() == [0, 9, 3, 3]
    with pytest.raises(IndexError):                      # CFG against a table without a null class
        solvers._check_labels(net, torch.tensor([1, 2, 10, 10]), 4, "cpu")
    with pytest.raises(ValueError):                      # a short label vector (dopri5 would read past its end)
        solvers._check_labels(net, torch.tensor([1, 2]), 4, "cpu")
    assert solvers._check_labels(net, None, 4, "cpu") is None
    edm = lfm_b200.DhariwalUNet(img_resolution=16, in_channels=4, out_channels=4, label_dim=5, model_channels=128,
                                channel_mult=(1, 2), num_blocks=1, attn_resolutions=(8,))
    with pytest.raises(RuntimeError):                    # one_hot semantics
        solvers._check_labels(edm, torch.tensor([0, 5]), 2, "cpu")
    edm0 = lfm_b200.DhariwalUNet(img_resolution=16, in_channels=4, out_channels=4, label_dim=0, model_channels=128,
                                 channel_mult=(1, 2), num_blocks=1, attn_resolutions=(8,))
    assert solvers._check_labels(edm0, torch.tensor([7]), 2, "cpu") is None   # no map_label: y is ignored (EDM.py:823)
    with pytest.raises(NotImplementedError):
        lfm_b200.UNetModel(image_size=32, in_channels=4, model_channels=128, out_channels=4, num_res_blocks=1,
                           attention_resolutions=(2,), channel_mult=(1, 2), num_heads=2, num_heads_upsample=4,
                           use_scale_shift_norm=True)


def test_vae_decoder_state_dict_surface():
    """lfm_b200.AutoencoderKL holds the decoder-side keys of the diffusers checkpoint (oracle.vae.param_shapes restates
    them), accepts a full / legacy-named checkpoint, and refuses to run on the CPU."""
    from oracle import vae as ovae
    vae = lfm_b200.AutoencoderKL()
    want = ovae.param_shapes(ovae.VAEConfig())
    got = {k: tuple(v.shape) for k, v in vae.state_dict().items()}
    assert got == want and len(got) == 140
    sd = lfm_b200.synthetic_vae_state_dict(vae, 3)
    ref = ovae.synthetic_state_dict(ovae.VAEConfig(), 3)
    assert all(torch.equal(sd[k], ref[k]) for k in ref)
    # a full checkpoint with the legacy attention names (what stabilityai/sd-vae-ft-mse ships) loads strictly
    legacy = {}
    for k, v in sd.items():
        for new, old in (("to_q", "query"), ("to_k", "key"), ("to_v", "value"), ("to_out.0", "proj_attn")):
            if f".attentions.0.{new}." in k:
                k = k.replace(f".{new}.", f".{old}.")
        legacy[k] = v
    legacy["encoder.conv_in.weight"] = torch.zeros(128, 3, 3, 3)
    legacy["quant_conv.weight"] = torch.zeros(8, 8, 1, 1)
    vae.load_state_dict(legacy, strict=True)
    assert torch.equal(vae.decoder.mid_block.attentions[0].to_out[0].weight, sd["decoder.mid_block.attentions.0.to_out.0.weight"])
    with pytest.raises(RuntimeError):
        bad = dict(sd)
        bad.pop("decoder.conv_out.bias")
        vae.load_state_dict(bad, strict=True)
    with pytest.raises(RuntimeError):                              # no CPU path
        vae.decode(torch.randn(1, 4, 32, 32))
    with pytest.raises(FileNotFoundError):                         # no hub access: only local directories
        lfm_b200.AutoencoderKL.from_pretrained("stabilityai/sd-vae-ft-mse")
    # post-processing restatement: truncation, not rounding (test_flow_latent_ddp.py:131-135)
    x = torch.tensor([[[[-1.5, -1.0, 0.0]], [[0.999, 1.0, 2.0]], [[0.2, 0.4, 0.6]]]])
    u = ovae.to_uint8_nhwc(x)
    assert u.shape == (1, 1, 3, 3) and u[0, 0, :, 0].tolist() == [0, 0, 127] and u[0, 0, :, 1].tolist() == [254, 255, 255]


def test_image_sink_writes_files_in_order(tmp_path):
    """The generation loop's file sink (lfm_b200.cli.ImageSink): batches handed over without blocking are all on disk
    after close(), each file holding its own image (decoded back and compared), buffers recycled across batches."""
    import numpy as np
    from PIL import Image
    from lfm_b200.cli import ImageSink
    sink = ImageSink(torch.device("cpu"), threads=3)
    want = {}
    g = torch.Generator().manual_seed(0)
    for b in range(5):
        u8 = (torch.rand(4, 1, 1, 3, generator=g) * 255).to(torch.uint8).expand(4, 16, 16, 3).contiguous()   # flat colours survive JPEG
        paths = [str(tmp_path / f"{b * 4 + j}.png") for j in range(4)]
        sink.put(u8, paths)
        for j, p in enumerate(paths):
            want[p] = u8[j].numpy().copy()
    sink.close()
    assert len(list(tmp_path.iterdir())) == 20
    for p, arr in want.items():
        assert np.array_equal(np.asarray(Image.open(p)), arr)
