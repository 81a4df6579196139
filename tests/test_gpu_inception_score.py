"""lfm_b200.inception_score on the GPU, with seeded stand-in Inception weights: the device against the CPU path, the
``--compute_fid --compute_is`` generation loop against the file command line on the same images, and two gloo ranks of
that loop against one process."""
import os

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from lfm_b200 import cli, fid
from lfm_b200 import inception_score as lis

DEV = "cuda:0"
LOOP = ["--model_type", "DiT-B/2", "--image_size", "256", "--num_in_channels", "4", "--num_classes", "1",
        "--label_dropout", "0.", "--method", "euler", "--step_size", "0.25", "--synthetic_init", "3", "--synthetic_vae", "2",
        "--device", DEV, "--dataset", "custom", "--exp", "t", "--compute_fid", "--compute_is", "--synthetic_inception", "1",
        "--no_save"]


def _weights(seed=1):
    return {**fid.synthetic_inception_state_dict(seed), **fid.synthetic_fc_state_dict(seed)}


def _u8(n, side, seed):
    return (torch.rand(n, side, side, 3, generator=torch.Generator().manual_seed(seed)) * 256).clamp_max(255).to(torch.uint8)


def _rel(a, b):
    return float(np.linalg.norm(np.asarray(a, dtype=np.float64) - b) / np.linalg.norm(b))


def _close(a, b, tol=1e-5):
    """(mean, std) pairs: each within ``tol`` of the mean (a one-split std is 0).  The stand-in network predicts nearly
    the same class for every image, so the scores sit just above 1 (1.0001 .. 1.002 on an H100); the part that depends
    on the images, ``log IS`` and the std, is also held to 1e-3 relative (1e-5 .. 1e-4 measured)."""
    return (abs(a[0] - b[0]) <= tol * abs(b[0]) and abs(a[1] - b[1]) <= tol * abs(b[0])
            and abs(np.log(a[0]) - np.log(b[0])) <= 1e-3 * abs(np.log(b[0])) and abs(a[1] - b[1]) <= 1e-3 * b[1] + 1e-12)


@pytest.fixture(scope="module")
def setup(tmp_path_factory):
    base = tmp_path_factory.mktemp("inception_score")
    weights = base / "stand_in.pth"
    torch.save(_weights(1), weights)
    stat = base / "stat.npy"           # the FID of the loop needs a statistics file; its value is not looked at here
    feats = np.random.RandomState(0).rand(64, 2048)
    np.save(stat, {"mu": feats.mean(0), "sigma": np.cov(feats, rowvar=False)}, allow_pickle=True)
    return base, str(weights), str(stat)


@pytest.mark.gpu
def test_device_agrees_with_cpu():
    net = fid.FIDInception(_weights(1), with_logits=True)
    net_gpu = fid.FIDInception(_weights(1), with_logits=True).to(DEV)
    for n, side, seed in ((24, 64, 1), (4, 256, 2)):
        u8 = _u8(n, side, seed)
        p_cpu = lis.inception_probs(net, u8)
        p_gpu = lis.inception_probs(net_gpu, u8.to(DEV)).cpu()
        rel = _rel(p_gpu.numpy(), p_cpu.numpy())
        print(f"{n} images of {side}^2: probabilities rel-L2 GPU vs CPU {rel:.3e}")
        assert rel <= 1e-5
        for splits in (1, 3):
            cpu, gpu = lis.ISStatistics(splits, n), lis.ISStatistics(splits, n, DEV)
            cpu.update(p_cpu, 0)
            gpu.update(p_gpu.to(DEV), 0)
            a, b = gpu.finalize(), cpu.finalize()
            print(f"  S = {splits}: IS GPU {a}, CPU {b}")
            assert _close(a, b)


def _log_is(path):
    line = [ln for ln in open(path).read().splitlines() if ", IS = " in ln][-1]
    mean, std = line.split("IS = ")[1].split(" +/- ")
    return float(mean), float(std)


def _file_cli(base, weights, images_nhwc, splits, tag):
    path = base / f"{tag}.npy"
    np.save(path, np.concatenate(images_nhwc, 0).transpose(0, 3, 1, 2))     # [N, 3, H, W] uint8, file-index order
    return lis.main(["--sample_dir", str(path), "--inception_weights", weights, "--splits", str(splits), "--device", DEV])


@pytest.mark.gpu
@pytest.mark.parametrize("splits", [1, 2])
def test_generation_loop_matches_the_file_cli(setup, splits, monkeypatch, capsys):
    base, weights, stat = setup
    seen = []
    probs = lis.inception_probs

    def capture(net, images, batch=64):
        seen.append(images.cpu().numpy())
        return probs(net, images, batch)
    monkeypatch.setattr(lis, "inception_probs", capture)
    log = base / f"loop_{splits}.log"
    assert cli.main(LOOP + ["--out_dir", str(base), "--batch_size", "3", "--n_sample", "6", "--is_splits", str(splits),
                            "--real_img_dir", stat, "--output_log", str(log)]) == 0
    monkeypatch.undo()
    out = capsys.readouterr().out
    lines = open(log).read().splitlines()
    assert lines[0].startswith("Epoch = 1000, FID = ") and lines[1].startswith("Epoch = 1000, IS = ")
    loop = _log_is(log)
    assert "IS = {} +/- {}".format(*loop) in out
    assert [a.shape for a in seen] == [(3, 256, 256, 3)] * 2
    ref = _file_cli(base, weights, seen, splits, f"loop_{splits}")
    print(f"S = {splits}: loop IS {loop}, file CLI {ref}")
    assert np.isfinite(loop[0]) and loop[0] > 1
    assert _close(loop, ref)


def _loop_rank(rank, world, port, argv, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from lfm_b200 import cli as c, inception_score as s
    seen, probs = [], s.inception_probs

    def capture(net, images, batch=64):
        seen.append(images.cpu().numpy())
        return probs(net, images, batch)
    s.inception_probs = capture
    rc = c.main(argv)
    q.put((rank, rc, seen))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.gpu
def test_two_gloo_ranks_give_the_one_process_number(setup):
    base, weights, stat = setup
    log = base / "two.log"
    argv = LOOP + ["--out_dir", str(base), "--batch_size", "3", "--n_sample", "12", "--is_splits", "3",
                   "--real_img_dir", stat, "--output_log", str(log)]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29700 + (os.getpid() % 90)
    procs = [ctx.Process(target=_loop_rank, args=(r, 2, port, argv, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=900) for _ in range(2)], key=lambda r: r[0])
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    assert [r[1] for r in res] == [0, 0]
    # image j of rank r's batch b is file index b * 6 + j * 2 + r: interleave the ranks back into index order
    batches = [np.stack([res[i % 2][2][b][i // 2] for i in range(6)]) for b in range(2)]
    two = _log_is(log)
    one = _file_cli(base, weights, batches, 3, "two_ranks")
    print(f"two gloo ranks: IS {two}; one process on the same images {one}")
    assert _close(two, one)
