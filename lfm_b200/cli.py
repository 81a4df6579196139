"""test_flow_latent.py-compatible sampling command line, running on liblfm_b200.so.

    python -m lfm_b200.cli --exp celeb_f8_dit --dataset celeba_256 --model_type DiT-L/2 --image_size 256 --f 8 \
        --num_in_channels 4 --num_out_channels 4 --num_classes 1 --label_dropout 0. --batch_size 64 \
        --method euler --step_size 0.02 --epoch_id 475

Same flags, defaults and modes as the reference (test_flow_latent.py:302-408): default "inference" (one batch ->
image grid), ``--compute_nfe``, ``--measure_time``, ``--compute_fid`` (generation loop with the reference's file
indexing; with ``--inception_weights FILE`` the FID itself is computed on the device from the decoded uint8 batches,
lfm_b200/fid.py, and printed / logged as the reference does, test_flow_latent.py:274-282).  Under
``torchrun`` (RANK/WORLD_SIZE set) it behaves like test_flow_latent_ddp.py: one process per GPU, per-rank batches,
seed = seed + rank, file index j * world + rank + total.

Differences, all deliberate (SURVEY.md Appendix B):
  * the Karras path works (the reference's CLI raises NameError / TypeError there);
  * ``--device`` exists; nothing is hard-coded to "cuda";
  * ``--synthetic_init SEED`` runs without a checkpoint (seeded non-degenerate weights);
  * ``--fp8`` (DiT only, off by default) runs the qkv and fc1 GEMMs on e4m3 operands, see lfm_b200.network.DiT;
  * the VAE decode runs natively (lfm_b200.AutoencoderKL: ``--pretrained_autoencoder_ckpt`` = a LOCAL diffusers
    directory, or ``--synthetic_vae SEED``); ``--vae diffusers`` keeps the reference's torch module when that package is
    installed; with neither, latents are saved (``--no_decode``);
  * in the generation loop (``--compute_fid``) the post-processing (clamp -> uint8 -> NHWC) is fused into the native
    decoder, the images leave the GPU through pinned buffers asynchronously and a thread pool encodes the JPEGs, so the
    GPU does not wait for PIL (the reference encodes on the main thread, test_flow_latent_ddp.py:131-139).
"""
from __future__ import annotations

import argparse
import math
import os

import numpy as np
import torch


def build_parser():
    p = argparse.ArgumentParser("flow-matching parameters")
    p.add_argument("--generator", type=str, default="determ", choices=["dummy", "determ", "determ-indiv"])
    p.add_argument("--seed", type=int, default=42)
    p.add_argument("--compute_fid", action="store_true", default=False)
    p.add_argument("--compute_nfe", action="store_true", default=False)
    p.add_argument("--measure_time", action="store_true", default=False)
    p.add_argument("--epoch_id", type=int, default=1000)
    p.add_argument("--n_sample", type=int, default=50000)
    p.add_argument("--model_type", type=str, default="adm")
    p.add_argument("--image_size", type=int, default=32)
    p.add_argument("--f", type=int, default=8)
    p.add_argument("--scale_factor", type=float, default=0.18215)
    p.add_argument("--num_in_channels", type=int, default=3)
    p.add_argument("--num_out_channels", type=int, default=3)
    p.add_argument("--nf", type=int, default=256)
    p.add_argument("--centered", action="store_false", default=True)
    p.add_argument("--resamp_with_conv", type=bool, default=True)
    p.add_argument("--num_res_blocks", type=int, default=2)
    p.add_argument("--num_heads", type=int, default=4)
    p.add_argument("--num_head_upsample", type=int, default=-1)
    p.add_argument("--num_head_channels", type=int, default=-1)
    p.add_argument("--attn_resolutions", nargs="+", type=int, default=(16,))
    p.add_argument("--ch_mult", nargs="+", type=int, default=(1, 2, 2, 2))
    p.add_argument("--label_dim", type=int, default=0)
    p.add_argument("--augment_dim", type=int, default=0)
    p.add_argument("--dropout", type=float, default=0.0)
    p.add_argument("--num_classes", type=int, default=None)
    p.add_argument("--label_dropout", type=float, default=0.0)
    p.add_argument("--cfg_scale", type=float, default=1.0)
    p.add_argument("--layout", action="store_true")
    p.add_argument("--use_origin_adm", action="store_true")
    p.add_argument("--use_scale_shift_norm", type=bool, default=True)
    p.add_argument("--resblock_updown", type=bool, default=False)
    p.add_argument("--use_new_attention_order", type=bool, default=False)
    p.add_argument("--pretrained_autoencoder_ckpt", type=str, default="stabilityai/sd-vae-ft-mse")
    p.add_argument("--output_log", type=str, default="")
    p.add_argument("--exp", default="experiment_cifar_default")
    p.add_argument("--real_img_dir", default="./pytorch_fid/cifar10_train_stat.npy")
    p.add_argument("--dataset", default="cifar10")
    p.add_argument("--num_steps", type=int, default=40)
    p.add_argument("--batch_size", type=int, default=200)
    p.add_argument("--use_karras_samplers", action="store_true", default=False)
    p.add_argument("--atol", type=float, default=1e-5)
    p.add_argument("--rtol", type=float, default=1e-5)
    p.add_argument("--method", type=str, default="dopri5",
                   choices=["dopri5", "dopri8", "adaptive_heun", "bosh3", "euler", "midpoint", "rk4", "heun", "multistep",
                            "stochastic", "dpm"])
    p.add_argument("--step_size", type=float, default=0.01)
    p.add_argument("--perturb", action="store_true", default=False)
    p.add_argument("--num_proc_node", type=int, default=1)
    p.add_argument("--num_process_per_node", type=int, default=1)
    p.add_argument("--node_rank", type=int, default=0)
    p.add_argument("--local_rank", type=int, default=0)
    p.add_argument("--master_address", type=str, default="127.0.0.1")
    p.add_argument("--master_port", type=str, default="6000")
    # additions
    p.add_argument("--device", type=str, default=None, help="cuda:N (default: cuda:LOCAL_RANK)")
    p.add_argument("--synthetic_init", type=int, default=None, metavar="SEED", help="seeded weights instead of a checkpoint")
    p.add_argument("--no_decode", action="store_true", help="skip the VAE decode; save latents (.npy)")
    p.add_argument("--vae", type=str, default="native", choices=["native", "diffusers"],
                   help="native: lfm_b200.AutoencoderKL (sm_90a kernels); diffusers: the reference's torch module")
    p.add_argument("--synthetic_vae", type=int, default=None, metavar="SEED", help="seeded decoder weights instead of a checkpoint")
    p.add_argument("--writer_threads", type=int, default=8, help="JPEG encoder threads of the --compute_fid loop")
    p.add_argument("--inception_weights", type=str, default=None, metavar="FILE",
                   help="local pt_inception-2015-12-05-6726825d.pth: compute the FID on the device in the --compute_fid loop")
    p.add_argument("--synthetic_inception", type=int, default=None, metavar="SEED",
                   help="seeded Inception weights (plumbing check only; the number is meaningless)")
    p.add_argument("--no_save", action="store_true", help="--compute_fid: do not write the JPEG files")
    p.add_argument("--out_dir", type=str, default=".")
    p.add_argument("--measure_reps", type=int, default=300)
    p.add_argument("--fp8", action="store_true", default=False,
                   help="DiT only: run the qkv and fc1 GEMMs on e4m3 operands (H100 FP8 tensor cores); results differ from bf16")
    return p


def load_model(args, device, ckpt_path=None):
    """create_network(args) with --synthetic_init weights, or the checkpoint at `ckpt_path` (default: the generation
    script's ./saved_info/latent_flow/... path) with its "module." prefix stripped."""
    from . import DhariwalUNet, UNetModel, create_network
    from .synthetic import synthetic_edm_state_dict, synthetic_state_dict, synthetic_unet_state_dict
    with torch.device("meta"):
        model = create_network(args)
    if args.synthetic_init is not None:
        make = (synthetic_unet_state_dict if isinstance(model, UNetModel)
                else synthetic_edm_state_dict if isinstance(model, DhariwalUNet) else synthetic_state_dict)
        sd = make(model, args.synthetic_init)
    else:
        path = ckpt_path or "./saved_info/latent_flow/{}/{}/model_{}.pth".format(args.dataset, args.exp, args.epoch_id)
        ckpt = torch.load(path, map_location="cpu")
        for key in list(ckpt.keys()):            # test_flow_latent.py:140-141 (strip "module.")
            ckpt[key[7:]] = ckpt.pop(key)
        sd = ckpt
    model = model.to_empty(device="cpu")
    model.load_state_dict(sd, strict=True)
    return model.to(device).eval()


_STAT_BY_DATASET = {      # test_flow_latent.py:113-126
    "cifar10": "cifar10_train_stat.npy", "celeba_256": "celebahq_stat.npy", "lsun_church": "lsun_church_stat.npy",
    "ffhq_256": "ffhq_stat.npy", "lsun_bedroom": "lsun_bedroom_stat.npy", "latent_imagenet_256": "imagenet_stat.npy",
    "imagenet_256": "imagenet_stat.npy",
}


def real_stats_path(args):
    """The dataset statistics file, chosen as the reference does (by --dataset, else --real_img_dir); when
    --real_img_dir names an existing file it wins, so the statistics need not live under ./pytorch_fid."""
    if os.path.isfile(args.real_img_dir):
        return args.real_img_dir
    if args.dataset in _STAT_BY_DATASET:
        return os.path.join("pytorch_fid", _STAT_BY_DATASET[args.dataset])
    return args.real_img_dir


def load_vae(args, device, with_encoder=False):
    """test_flow_latent.py:131 ``AutoencoderKL.from_pretrained(args.pretrained_autoencoder_ckpt).to(device)``; the
    native module holds the encoder too with `with_encoder`."""
    if args.no_decode:
        return None
    if args.vae == "diffusers":
        try:
            from diffusers.models import AutoencoderKL as TorchVAE
        except ImportError:
            raise SystemExit("--vae diffusers: the diffusers package is not installed (use the native decoder)")
        return TorchVAE.from_pretrained(args.pretrained_autoencoder_ckpt).to(device)
    from .vae import AutoencoderKL, synthetic_vae_state_dict
    if args.synthetic_vae is not None:
        vae = AutoencoderKL(with_encoder=with_encoder)
        vae.load_state_dict(synthetic_vae_state_dict(vae, args.synthetic_vae), strict=True)
        return vae.to(device).eval()
    if os.path.isdir(args.pretrained_autoencoder_ckpt):
        return AutoencoderKL.from_pretrained(args.pretrained_autoencoder_ckpt, with_encoder=with_encoder).to(device)
    print(f"'{args.pretrained_autoencoder_ckpt}' is not a local diffusers directory (no hub access here) and no "
          "--synthetic_vae seed was given: skipping the VAE decode, saving latents instead (--no_decode)")
    args.no_decode = True
    return None


class ImageSink:
    """Device -> pinned host -> JPEG files without stalling the sampler (test_flow_latent_ddp.py:131-139 does
    ``.to("cpu")`` + ``Image.fromarray(x).save`` per image on the main thread).  ``put`` enqueues an asynchronous D2H
    copy of a uint8 NHWC batch on a side stream and returns; a pool of encoder threads waits for the copy's event and
    writes the files.  Two pinned buffers alternate: the sampler is blocked only if it runs two batches ahead."""

    def __init__(self, device, threads=8):
        from concurrent.futures import ThreadPoolExecutor
        self.device = device
        self.pool = ThreadPoolExecutor(max_workers=max(1, threads))
        self.copy_stream = torch.cuda.Stream(device) if device.type == "cuda" else None
        self.bufs, self.pending, self.turn = [None, None], [[], []], 0

    def put(self, u8, paths):
        i = self.turn
        self.turn ^= 1
        for f in self.pending[i]:          # the buffer's previous batch must be on disk before it is overwritten
            f.result()
        if self.bufs[i] is None or self.bufs[i].shape != u8.shape:
            self.bufs[i] = torch.empty(u8.shape, dtype=torch.uint8, pin_memory=self.device.type == "cuda")
        host = self.bufs[i]
        if self.copy_stream is not None:
            ready = torch.cuda.Event()
            ready.record(torch.cuda.current_stream(self.device))
            with torch.cuda.stream(self.copy_stream):
                self.copy_stream.wait_event(ready)
                host.copy_(u8, non_blocking=True)
                done = torch.cuda.Event()
                done.record(self.copy_stream)
            u8.record_stream(self.copy_stream)
        else:
            host.copy_(u8)
            done = None
        arr = host.numpy()

        def write(j, path):
            if done is not None:
                done.synchronize()
            from PIL import Image
            Image.fromarray(arr[j]).save(path)
        self.pending[i] = [self.pool.submit(write, j, pth) for j, pth in enumerate(paths)]

    def close(self):
        for lst in self.pending:
            for f in lst:
                f.result()
        self.pool.shutdown(wait=True)


def make_run_sampling(args, model, vae, device):
    """test_flow_latent.py:161-194 / test_flow_latent_ddp.py:83-111."""
    from .solvers import sample_from_model, sample_from_model_with_fixed_step_solver

    def run_sampling(num_samples, generator, cls_index=None, return_nfe=False, as_uint8=False):
        side = args.image_size // 8
        x = generator.randn(num_samples, 4, side, side).to(device)
        if args.num_classes in [None, 1]:
            model_kwargs = {}
        else:
            if cls_index is None:
                y = generator.randint(0, args.num_classes, (num_samples,), device=device)
            else:
                y = torch.full((num_samples,), cls_index, device=device, dtype=torch.long)
            if args.cfg_scale > 1.0:
                x = torch.cat([x, x], 0)
                y_null = (torch.full((num_samples,), args.num_classes, device=device, dtype=torch.long)
                          if "DiT" in args.model_type else torch.zeros_like(y))
                model_kwargs = dict(y=torch.cat([y, y_null], 0), cfg_scale=args.cfg_scale)
            else:
                model_kwargs = dict(y=y)
        nfe = None
        if not args.use_karras_samplers:
            out = sample_from_model(model, x, model_kwargs, args)
            if args.compute_nfe:
                out, nfe = out
            fake_sample = out[-1]
        else:
            fake_sample = sample_from_model_with_fixed_step_solver(model, x, model_kwargs, generator, args)
            nfe = model.last_stats["nfe"]
        if args.cfg_scale > 1.0:
            fake_sample, _ = fake_sample.chunk(2, dim=0)
        if vae is None:
            result = fake_sample
        elif as_uint8 and hasattr(vae, "decode_to_uint8"):
            result = vae.decode_to_uint8(fake_sample / args.scale_factor)     # [n, H, W, 3] uint8, post-processing fused
        else:
            result = vae.decode(fake_sample / args.scale_factor).sample
        return (result, nfe) if return_nfe else result

    return run_sampling


def main(argv=None):
    args = build_parser().parse_args(argv)
    from . import dist as ldist
    from .random_util import get_generator

    rank, world, local = ldist.init_from_env()
    args.world_size = world
    torch.set_grad_enabled(False)
    seed = ldist.rank_seed(args.seed, rank)
    torch.manual_seed(seed)
    device = torch.device(args.device if args.device else f"cuda:{local}")
    if device.type == "cuda":
        torch.cuda.set_device(device)
        torch.cuda.manual_seed_all(seed)
    model = load_model(args, device)
    vae = load_vae(args, device)
    if rank == 0:
        print("Finish loading model; parameters: %.2f M" % (sum(p.numel() for p in model.parameters()) / 1e6))
    generator = get_generator(args.generator, args.n_sample, seed)
    run_sampling = make_run_sampling(args, model, vae, device)
    save_dir = os.path.join(args.out_dir, "generated_samples", args.dataset,
                            "exp{}_ep{}_m{}".format(args.exp, args.epoch_id, args.method))
    if args.use_karras_samplers or args.method in ("euler", "rk4", "midpoint", "stochastic"):
        save_dir += "_s{}".format(args.num_steps)

    if args.compute_nfe:
        was = args.compute_nfe
        total, trials = 0.0, min(300, args.measure_reps)
        for _ in range(trials):
            _, nfe = run_sampling(1, generator, return_nfe=True)
            total += float(nfe) / trials
        args.compute_nfe = was
        print(f"Average NFE over {trials} trials: {int(total)}")
        return 0

    if args.measure_time:
        side = args.image_size // 8
        x = generator.randn(1, 4, side, side).to(device)
        for _ in range(10):
            model(torch.tensor(1.0, device=device), x)
        timings = []
        for _ in range(args.measure_reps):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            run_sampling(1, generator)
            e.record()
            torch.cuda.synchronize()
            timings.append(s.elapsed_time(e))
        print("Inference time: {:.2f}+/-{:.2f}ms".format(float(np.mean(timings)), float(np.std(timings))))
        return 0

    if args.compute_fid:
        n = args.batch_size
        total_samples = ldist.total_samples(args.n_sample, n, world)
        iters = total_samples // world // n
        if rank == 0:
            os.makedirs(save_dir, exist_ok=True)
            print(f"Total number of images that will be sampled: {total_samples}")
        if world > 1:
            torch.distributed.barrier()
        total = 0
        sink = ImageSink(device, args.writer_threads) if vae is not None and not args.no_save else None
        fid_acc = None
        if args.inception_weights is not None or args.synthetic_inception is not None:
            if vae is None:
                raise ValueError("the FID needs decoded images: drop --no_decode")
            from . import fid as lfid
            net = (lfid.FIDInception.from_file(args.inception_weights) if args.inception_weights is not None
                   else lfid.FIDInception(lfid.synthetic_inception_state_dict(args.synthetic_inception)))
            fid_acc = lfid.FIDAccumulator(net, device)
        for i in range(iters):
            out = run_sampling(n, generator, as_uint8=True)
            if vae is None:
                for j, z in enumerate(out):
                    np.save("{}/{}.npy".format(save_dir, ldist.file_index(j, world, rank, total)), z.cpu().numpy())
            else:
                if out.dtype != torch.uint8:      # the torch VAE: the reference's expression (test_flow_latent_ddp.py:131-135)
                    out = (torch.clamp((out + 1.0) / 2.0, 0, 1) * 255.0).permute(0, 2, 3, 1).to(torch.uint8)
                if fid_acc is not None:
                    fid_acc.update(out)           # features + running statistics on the device; no file round trip
                if sink is not None:
                    sink.put(out, ["{}/{}.jpg".format(save_dir, ldist.file_index(j, world, rank, total))
                                   for j in range(out.shape[0])])
            total += n * world
            if rank == 0:
                print("generating batch ", i)
        if sink is not None:
            sink.close()
        if world > 1:
            torch.distributed.barrier()
        if fid_acc is not None:
            value = fid_acc.compute(real_stats_path(args))       # one all-reduce of the statistics across the ranks
            if rank == 0:
                print("FID = {}".format(value))                   # test_flow_latent.py:280-282
                if args.output_log:
                    with open(args.output_log, "a") as f:
                        f.write("Epoch = {}, FID = {}\n".format(args.epoch_id, value))
        elif rank == 0:
            print("samples written to", save_dir, "- pass --inception_weights FILE for the FID, or run pytorch_fid on them")
        return 0

    # default: one batch; every rank samples (and decodes) its shard and ONE all-gather assembles the result on all
    # ranks - of the decoded uint8 images when the native decoder runs (196 KB per 256 x 256 image, 768 KB at 512), else of the latents
    out = run_sampling(args.batch_size, generator, as_uint8=True)
    out = ldist.all_gather_batch(out)
    if rank == 0:
        if args.use_karras_samplers:
            stem = "samples_{}_{}_{}".format(args.dataset, args.method, args.num_steps)
        else:
            stem = "samples_{}_{}_{}_{}".format(args.dataset, args.method, args.atol, args.rtol)
        if args.num_classes is not None and args.num_classes > 1:
            stem += "_cfg{}".format(args.cfg_scale)
        os.makedirs(args.out_dir, exist_ok=True)
        if vae is None:
            path = os.path.join(args.out_dir, stem + "_latents.npy")
            np.save(path, out.cpu().numpy())
        else:
            import torchvision
            path = os.path.join(args.out_dir, stem + ".jpg")
            img = out.permute(0, 3, 1, 2).float() / 255.0 if out.dtype == torch.uint8 else torch.clamp((out + 1.0) / 2.0, 0, 1)
            torchvision.utils.save_image(img, path, padding=0, nrow=8)
        print("Samples are save at '{}".format(path))
    if world > 1:
        torch.distributed.barrier()
        torch.distributed.destroy_process_group()
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
