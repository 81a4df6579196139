"""lfm_b200.inception_score on the CPU: the split sums against the reference's ``preds2score`` and the logits against the
reference's network (tests/golden/is_ref.npz, oracle/make_is_goldens.py), the TF1 resize against its numpy restatement
(tests/tools/inception_score_oracle.py), the file command line, its refusals, and the all-reduce across gloo ranks."""
import os

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp
from PIL import Image

from lfm_b200 import cli, fid
from lfm_b200 import inception_score as lis
from tests.tools.inception_score_oracle import prepare_reference

GOLD = os.path.join(os.path.dirname(__file__), "golden", "is_ref.npz")


def _inputs():
    g = torch.Generator().manual_seed(11)          # oracle/make_is_goldens.py:seeded_inputs
    return torch.rand(2, 3, 299, 299, generator=g) * 2 - 1


def _weights(seed=1):
    return {**fid.synthetic_inception_state_dict(seed), **fid.synthetic_fc_state_dict(seed)}


def _u8(n, side, seed):
    return (torch.rand(n, side, side, 3, generator=torch.Generator().manual_seed(seed)) * 256).clamp_max(255).to(torch.uint8)


def _rel(a, b):
    return float(np.linalg.norm(np.asarray(a, dtype=np.float64) - b) / np.linalg.norm(b))


@pytest.fixture(scope="module")
def net():
    return fid.FIDInception(_weights(1), with_logits=True)


@pytest.fixture(scope="module")
def weight_file(tmp_path_factory):
    path = tmp_path_factory.mktemp("is_weights") / "stand_in.pth"
    torch.save(_weights(1), path)
    return str(path)


@pytest.mark.parametrize("n", [37, 100])
@pytest.mark.parametrize("splits", [1, 3, 10])
def test_split_sums_match_reference_preds2score(n, splits):
    z = np.load(GOLD)
    st = lis.ISStatistics(splits, n)
    st.update(torch.from_numpy(z[f"probs_{n}"]), 0)
    mean, std = st.finalize()
    ref_mean, ref_std = float(z[f"mean_{n}_{splits}"]), float(z[f"std_{n}_{splits}"])
    assert abs(mean - ref_mean) <= 1e-6 * ref_mean                  # the reference sums in fp32; 2e-7 measured
    assert abs(std - ref_std) <= 1e-6 * ref_mean


@pytest.mark.parametrize("chunk", [1, 7, 100])
def test_chunked_updates_give_the_same_sums(chunk):
    p = torch.from_numpy(np.load(GOLD)["probs_100"])
    whole = lis.ISStatistics(10, 100)
    whole.update(p, 0)
    parts = lis.ISStatistics(10, 100)
    for i in range(0, 100, chunk):
        parts.update(p[i:i + chunk], i)
    assert torch.allclose(parts.buf, whole.buf, rtol=1e-13, atol=0)
    assert abs(parts.finalize()[0] - whole.finalize()[0]) < 1e-12 * whole.finalize()[0]


@pytest.mark.parametrize("n, splits", [(50000, 10), (37, 4), (37, 10), (100, 3)])
def test_split_of_index_is_the_reference_slice(n, splits):
    ref = np.empty(n, dtype=np.int64)
    for i in range(splits):                        # inception_score.py:85
        ref[i * n // splits:(i + 1) * n // splits] = i
    got = lis.ISStatistics(splits, n).split_of(torch.arange(n)).numpy()
    assert np.array_equal(got, ref)


@pytest.mark.parametrize("side", [32, 64, 256, 299, 512])
def test_prepare_tf1_matches_the_restated_resize(side):
    u8 = _u8(2, side, side)
    got = lis.prepare_tf1(u8)
    assert got.shape == (2, 3, 299, 299) and got.dtype == torch.float32
    ref = prepare_reference(u8.permute(0, 3, 1, 2).numpy())
    assert np.abs(got.numpy() - ref).max() <= 1e-6                 # /255 in fp32 here, in fp64 there: 1 ulp
    assert torch.equal(lis.prepare_tf1(u8.permute(0, 3, 1, 2).float()), got)     # float NCHW in 0..255: the same path
    if side == 299:
        assert torch.equal(got, u8.permute(0, 3, 1, 2).float() / 255.0 * 2 - 1)  # identity resize


def test_prepare_tf1_refuses_bad_layouts():
    with pytest.raises(ValueError):
        lis.prepare_tf1(torch.zeros(2, 3, 32, 32, dtype=torch.uint8))           # uint8 must be NHWC
    with pytest.raises(ValueError):
        lis.prepare_tf1(torch.zeros(2, 32, 32, 3))                                # float must be NCHW


def test_logits_match_the_reference_network(net):
    z = np.load(GOLD)
    logits = net.logits(_inputs())
    assert logits.shape == (2, 1008)
    assert _rel(logits.numpy(), z["logits"]) <= 1e-5                # 3e-7 measured


def test_fid_features_unchanged_with_fc():
    u8 = _u8(2, 48, 3)
    plain = fid.FIDInception(fid.synthetic_inception_state_dict(1))
    with_fc = fid.FIDInception(_weights(1), with_logits=True)
    ignored = fid.FIDInception(_weights(1))                        # fc.* present but not asked for
    f = plain(u8)
    assert torch.equal(with_fc(u8), f) and torch.equal(ignored(u8), f)
    assert torch.equal(plain.trunk(fid.FIDInception.prepare(u8)), f)
    with pytest.raises(RuntimeError):
        plain.logits(_inputs())


def test_fc_is_loaded_strictly_when_asked_for():
    with pytest.raises(ValueError, match="fc"):
        fid.FIDInception(fid.synthetic_inception_state_dict(1), with_logits=True)
    bad = _weights(1)
    bad["fc.weight"] = torch.zeros(1000, 2048)
    with pytest.raises(ValueError):
        fid.FIDInception(bad, with_logits=True)
    assert {k: tuple(v.shape) for k, v in fid.synthetic_fc_state_dict(1).items()} == fid.FC_SHAPES
    assert len(fid.synthetic_inception_state_dict(1)) == 94 * 5


def test_statistics_refusals():
    with pytest.raises(ValueError):
        lis.ISStatistics(0, 10)
    with pytest.raises(ValueError):
        lis.ISStatistics(11, 10)
    st = lis.ISStatistics(2, 10)
    with pytest.raises(ValueError):
        st.update(torch.full((3, 1008), 1e-3), 0)
    with pytest.raises(ValueError):
        st.update(torch.full((3, 1000), 1e-3), 8)                     # indices 8..10 of 10 images
    st.update(torch.full((5, 1000), 1e-3), 0)
    with pytest.raises(ValueError):
        st.finalize()                                                 # split 1 has no image yet


def test_parser_defaults():
    a = lis.build_parser().parse_args(["--inception_weights", "w.pth"])
    assert (a.sample_dir, a.splits, a.batch_size, a.device) == ("./saved_samples/", 1, 64, None)
    c = cli.build_parser().parse_args([])
    assert c.compute_is is False and c.is_splits == 10


def test_cli_refuses_is_outside_the_generation_loop():
    with pytest.raises(ValueError, match="--compute_fid"):
        cli.main(["--compute_is", "--synthetic_inception", "1"])


def test_file_cli_refusals(tmp_path, weight_file):
    def run(arr, *extra, weights=weight_file):
        np.save(tmp_path / "x.npy", arr)
        return lis.main(["--sample_dir", str(tmp_path / "x.npy"), "--inception_weights", weights, "--device", "cpu", *extra])
    good = np.full((4, 3, 16, 16), 128, dtype=np.uint8)
    with pytest.raises(ValueError, match="N, 3, H, W"):
        run(good[0])                                                  # rank 3
    with pytest.raises(ValueError, match="N, 3, H, W"):
        run(good.transpose(0, 2, 3, 1))                               # channels last
    with pytest.raises(ValueError, match="range"):
        run(good / 255.0)                                             # scaled to [0, 1]
    with pytest.raises(ValueError):
        run(good, "--splits", "0")
    with pytest.raises(ValueError, match="splits"):
        run(good, "--splits", "5")
    no_fc = tmp_path / "no_fc.pth"
    torch.save(fid.synthetic_inception_state_dict(1), no_fc)
    with pytest.raises(ValueError, match="fc"):
        run(good, weights=str(no_fc))
    with pytest.raises(RuntimeError):
        lis.main(["--sample_dir", str(tmp_path / "missing.npy"), "--inception_weights", weight_file])


def test_directory_order_rule(tmp_path):
    for name in ("10.png", "2.png", "1.jpg"):
        Image.new("RGB", (4, 4)).save(tmp_path / name)
    assert [f.name for f in lis.list_images_in_order(str(tmp_path))] == ["1.jpg", "2.png", "10.png"]
    Image.new("RGB", (4, 4)).save(tmp_path / "a.png")
    assert [f.name for f in lis.list_images_in_order(str(tmp_path))] == ["1.jpg", "10.png", "2.png", "a.png"]


def _expected(net, images_u8, splits):
    st = lis.ISStatistics(splits, images_u8.shape[0])
    st.update(lis.inception_probs(net, images_u8), 0)
    return st.finalize()


def test_npy_path_clips_and_scores(tmp_path, weight_file, net, capsys):
    u8 = _u8(5, 24, 9)
    arr = u8.permute(0, 3, 1, 2).numpy().astype(np.float32)
    arr[:, :, :4] = np.where(arr[:, :, :4] > 128, 300.0, -40.0)      # out-of-range values: clipped to 0 / 255
    np.save(tmp_path / "x.npy", arr)
    mean, std = lis.main(["--sample_dir", str(tmp_path / "x.npy"), "--inception_weights", weight_file,
                          "--splits", "2", "--batch-size", "2", "--device", "cpu"])
    clipped = torch.from_numpy(np.clip(arr, 0, 255)).to(torch.uint8).permute(0, 2, 3, 1)
    ref_mean, ref_std = _expected(net, clipped, 2)
    assert abs(mean - ref_mean) < 1e-5 * ref_mean and abs(std - ref_std) < 1e-5 * ref_mean
    out = capsys.readouterr().out.splitlines()
    assert out[-3] == "Calculating Inception Score with 5 images in 2 splits"
    assert out[-2].startswith("mean:  ") and out[-1].startswith("std:  ")


def test_directory_path_scores_in_index_order(tmp_path, weight_file, net):
    u8 = _u8(4, 20, 4)
    for k in range(4):
        Image.fromarray(u8[k].numpy()).save(tmp_path / f"{k * 5}.png")      # 0, 5, 10, 15: name order is 0, 10, 15, 5
    mean, std = lis.main(["--sample_dir", str(tmp_path), "--inception_weights", weight_file, "--splits", "2",
                          "--device", "cpu"])
    ref_mean, ref_std = _expected(net, u8, 2)
    assert abs(mean - ref_mean) < 1e-5 * ref_mean and abs(std - ref_std) < 1e-5 * ref_mean
    Image.new("RGB", (8, 8)).save(tmp_path / "20.png")
    with pytest.raises(ValueError, match="differ in size"):
        lis.main(["--sample_dir", str(tmp_path), "--inception_weights", weight_file, "--device", "cpu"])


def _rank_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    net = fid.FIDInception(_weights(1), with_logits=True)
    images = _u8(6, 16, 21)
    st = lis.ISStatistics(3, 6)
    st.update(lis.inception_probs(net, images[rank::world]), rank, world)   # the loop's file index j * world + rank
    st.all_reduce()
    q.put((rank, st.buf.numpy(), st.finalize()))
    dist.barrier()
    dist.destroy_process_group()


def test_two_gloo_ranks_reduce_to_one_process(net):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29800 + (os.getpid() % 90)
    procs = [ctx.Process(target=_rank_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in range(2)]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    one = lis.ISStatistics(3, 6)
    one.update(lis.inception_probs(net, _u8(6, 16, 21)), 0)
    for _, buf, (mean, std) in res:
        assert np.allclose(buf, one.buf.numpy(), rtol=1e-6, atol=1e-9)
        ref_mean, ref_std = one.finalize()
        assert abs(mean - ref_mean) < 1e-6 * ref_mean and abs(std - ref_std) < 1e-6 * ref_mean
