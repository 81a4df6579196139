"""Semantic-synthesis (mask-to-image) command line (downstream_tasks/test_flow_latent_semantic_syn.py), running on
liblfm_b200.so.

    python test_flow_latent_semantic_syn.py --exp semantic_kl --dataset celeba --epoch_id 175 --batch_size 64 \
        --attn_resolution 16 8 --method dopri5 --pretrained_autoencoder_ckpt ./sd-vae-ft-mse

Same flags and defaults as the reference (test_flow_latent_semantic_syn.py:154-229), the segmentation semantics of its
``CelebAMaskValidation`` and its checkpoints, ``./saved_info/latent_flow_mask2image/{dataset}/{exp}/model_{epoch}.pth`` and
``cond_stage_model_{epoch}.pth``, both with the "module." prefix stripped.  Per batch: the uint8 label maps go to the device,
``SpatialRescaler.forward_labels`` turns them into the 4-channel condition of the 8-channel UNetModel in one kernel (the
reference's one-hot, three bilinear halvings and 1x1 conv), the solver runs ``WrapperCondFlow(model, c)`` from
``z_0 ~ N(0, I)``, the result is decoded and mapped to [0, 1], and written as ``{index}.jpg`` under
``{out_dir}/mask2image_generated_samples/{dataset}/``.  Condition, UNet, solver and decoder all run natively.

Only ``--dataset celeba`` (19 classes) is supported: the reference's ADE20k and COCO readers are not, and for any other value
(its default ``cifar10``, or the readme's ``celeba_256``) the reference itself fails with ``dataset`` unbound.

Differences, all deliberate:
  * the paths the reference hard-codes are flags with its values as defaults: ``--mask_dir``, ``--num_images`` (its dataset
    length), ``--out_dir``; ``--num_workers`` is its DataLoader's 4;
  * ``--synthetic_init SEED`` (seeded UNet weights, and a ``channel_mapper`` weight drawn as ``N(0, 1) / sqrt(19)``),
    ``--synthetic_vae SEED`` and ``--device`` as in lfm_b200.cli;
  * only the segmentation maps are read: the reference also loads and resizes each 1024-pixel image, only to take its batch
    size;
  * the reference calls ``save_image(x, path, normalized=True)``, which raises TypeError on current torchvision (make_grid has
    no ``normalized`` argument); the files here hold what ``save_image(x, path)`` writes, ``(x * 255 + 0.5).clamp(0, 255)`` as uint8;
  * the CPU and CUDA generators are seeded with ``--seed`` (the reference seeds 42 and ignores it); ``z_0`` is drawn on the CPU
    as there, but its stream is not the reference's, which also depends on module initialisation and DataLoader worker seeding;
  * ``index`` is the running image count ``i * batch_size + j``; the reference writes ``i * image.size(0) + j``, which
    overwrites earlier files when the last batch is partial.
"""
from __future__ import annotations

import argparse
import os
import types

import numpy as np
import torch

from . import cli

NUM_CLASSES = {"celeba": 19}          # test_flow_latent_semantic_syn.py:88-94; ADE20k (151) and COCO (182) are not read here
FIRST_VALIDATION_INDEX = 27000        # CelebAMask-HQ: the first 27000 images train, the next 3000 validate
SIZE = 256


def build_parser():
    p = argparse.ArgumentParser("ddgan parameters")
    p.add_argument("--seed", type=int, default=1024)
    p.add_argument("--compute_fid", action="store_true", default=False)
    p.add_argument("--epoch_id", type=int, default=425)
    p.add_argument("--image_size", type=int, default=256)
    p.add_argument("--num_in_channels", type=int, default=8)
    p.add_argument("--num_out_channels", type=int, default=4)
    p.add_argument("--nf", type=int, default=256)
    p.add_argument("--centered", action="store_false", default=True)
    p.add_argument("--resamp_with_conv", type=bool, default=True)
    p.add_argument("--num_res_blocks", type=int, default=2)
    p.add_argument("--num_heads", type=int, default=4)
    p.add_argument("--num_head_upsample", type=int, default=-1)
    p.add_argument("--num_head_channels", type=int, default=-1)
    p.add_argument("--attn_resolutions", nargs="+", type=int, default=(8, 4))
    p.add_argument("--ch_mult", nargs="+", type=int, default=(1, 2, 3, 4))
    p.add_argument("--dropout", type=float, default=0.0)
    p.add_argument("--num_classes", type=int, default=None)
    p.add_argument("--use_scale_shift_norm", type=bool, default=True)
    p.add_argument("--resblock_updown", type=bool, default=False)
    p.add_argument("--use_new_attention_order", type=bool, default=False)
    p.add_argument("--scale_factor", type=float, default=0.18215)
    p.add_argument("--exp", default="experiment_cifar_default")
    p.add_argument("--real_img_dir", default="./pytorch_fid/cifar10_train_stat.npy")
    p.add_argument("--dataset", default="cifar10")
    p.add_argument("--num_timesteps", type=int, default=200)
    p.add_argument("--batch_size", type=int, default=200)
    p.add_argument("--atol", type=float, default=1e-5)
    p.add_argument("--rtol", type=float, default=1e-5)
    p.add_argument("--method", type=str, default="dopri5",
                   choices=["dopri5", "dopri8", "adaptive_heun", "bosh3", "euler", "midpoint", "rk4"])
    p.add_argument("--step_size", type=float, default=0.01)
    p.add_argument("--perturb", action="store_true", default=False)
    p.add_argument("--pretrained_autoencoder_ckpt", type=str, default="../stabilityai/sd-vae-ft-mse")
    # additions
    p.add_argument("--mask_dir", type=str, default="dataset/CelebAMask-HQ/mask", help="label maps {27000 + i}.png")
    p.add_argument("--num_images", type=int, default=3000, help="images of the evaluation set")
    p.add_argument("--num_workers", type=int, default=4, help="DataLoader workers")
    p.add_argument("--out_dir", type=str, default=".")
    p.add_argument("--device", type=str, default=None, help="cuda:N (default: cuda:0)")
    p.add_argument("--synthetic_init", type=int, default=None, metavar="SEED",
                   help="seeded UNet and channel_mapper weights instead of checkpoints")
    p.add_argument("--synthetic_vae", type=int, default=None, metavar="SEED", help="seeded VAE weights instead of a checkpoint")
    return p


def parse_args(argv=None):
    """build_parser().parse_args, and the refusal of a dataset without a reader here."""
    p = build_parser()
    args = p.parse_args(argv)
    if args.dataset not in NUM_CLASSES:
        p.error(f"--dataset {args.dataset}: 'celeba' (CelebAMask-HQ, 19 classes) is the supported dataset")
    return args


def resize_nearest(seg):
    """albumentations ``SmallestMaxSize(256, cv2.INTER_NEAREST)`` then ``CenterCrop(256)`` of a square [S, S] map: output
    pixel d takes source pixel floor(d S / 256) along each axis (cv2's nearest rule; S / 256 is exact in binary)."""
    S = seg.shape[0]
    idx = (np.arange(SIZE) * S) // SIZE
    return seg[idx[:, None], idx[None, :]]


class CelebAMaskSegmentation(torch.utils.data.Dataset):
    """The segmentation half of ``CelebAMaskValidation(size=256, crop_size=256)``: item i is ``{mask_dir}/{27000 + i}.png``
    as a uint8 [256, 256] label map.  Maps that are not 2-D or not square, or hold labels >= num_classes, are refused with
    ValueError naming the file."""

    def __init__(self, mask_dir, length=3000, num_classes=19):
        self.mask_dir, self.length, self.num_classes = mask_dir, length, num_classes

    def __len__(self):
        return self.length

    def path(self, i):
        return os.path.join(self.mask_dir, "{}.png".format(FIRST_VALIDATION_INDEX + i))

    def __getitem__(self, i):
        from PIL import Image
        path = self.path(i)
        seg = np.array(Image.open(path))
        if seg.ndim != 2 or seg.shape[0] != seg.shape[1]:
            raise ValueError(f"{path}: a label map must be a square single-channel image, got shape {seg.shape}")
        if int(seg.min()) < 0 or int(seg.max()) >= self.num_classes:
            raise ValueError(f"{path}: labels must lie in [0, {self.num_classes}), got values in [{int(seg.min())}, {int(seg.max())}]")
        return torch.from_numpy(np.ascontiguousarray(resize_nearest(seg.astype(np.uint8))))


def _load_stripped(path):
    ckpt = torch.load(path, map_location="cpu")
    for key in list(ckpt.keys()):             # test_flow_latent_semantic_syn.py:101-102, 117-118 (strip "module.")
        ckpt[key[7:]] = ckpt.pop(key)
    return ckpt


def load(args, device):
    """The 8-channel UNetModel (get_flow_model), the SpatialRescaler(n_stages=3, 19 -> 4) condition stage and the AutoencoderKL
    decoder, all loaded strictly."""
    from .downstream import SpatialRescaler
    if args.synthetic_vae is None and not os.path.isdir(args.pretrained_autoencoder_ckpt):
        raise SystemExit(f"'{args.pretrained_autoencoder_ckpt}' is not a local diffusers directory (no hub access here): "
                         "pass a local copy or --synthetic_vae SEED")
    num_cls = NUM_CLASSES[args.dataset]
    root = "./saved_info/latent_flow_mask2image/{}/{}".format(args.dataset, args.exp)
    cond = SpatialRescaler(n_stages=3, in_channels=num_cls, out_channels=4, multiplier=0.5)
    if args.synthetic_init is not None:
        g = torch.Generator().manual_seed(args.synthetic_init)
        sd = {"channel_mapper.weight": torch.randn(4, num_cls, 1, 1, generator=g) / num_cls ** 0.5}
    else:
        sd = _load_stripped(os.path.join(root, "cond_stage_model_{}.pth".format(args.epoch_id)))
    cond.load_state_dict(sd, strict=True)
    cond = cond.to(device).eval()
    margs = types.SimpleNamespace(**vars(args), use_origin_adm=True, layout=False)
    model = cli.load_model(margs, device, ckpt_path=os.path.join(root, "model_{}.pth".format(args.epoch_id)))
    vargs = types.SimpleNamespace(no_decode=False, vae="native", synthetic_vae=args.synthetic_vae,
                                  pretrained_autoencoder_ckpt=args.pretrained_autoencoder_ckpt)
    return model, cond, cli.load_vae(vargs, device)


def synthesize(args, model, cond_stage_model, vae, seg):
    """One batch of test_flow_latent_semantic_syn.py:131-152 on the device: [B, H, W] uint8 label maps -> the generated
    images as uint8 NHWC [B, 8s, 8s, 3] (what save_image writes)."""
    from .downstream import WrapperCondFlow, sample_from_model
    device = seg.device
    c = cond_stage_model.forward_labels(seg)
    z_0 = torch.randn(seg.size(0), 4, args.image_size // 8, args.image_size // 8).to(device)
    fake_sample = sample_from_model(WrapperCondFlow(model, c), z_0, args)[-1]
    fake_image = (vae.decode(fake_sample / args.scale_factor).sample + 1.0) / 2.0
    return fake_image.mul(255).add_(0.5).clamp_(0, 255).permute(0, 2, 3, 1).to(torch.uint8)


def main(argv=None):
    args = parse_args(argv)
    torch.set_grad_enabled(False)
    device = torch.device(args.device if args.device else "cuda:0")
    torch.manual_seed(args.seed)
    if device.type == "cuda":
        torch.cuda.set_device(device)
        torch.cuda.manual_seed_all(args.seed)
    dataset = CelebAMaskSegmentation(args.mask_dir, args.num_images, NUM_CLASSES[args.dataset])
    loader = torch.utils.data.DataLoader(dataset, batch_size=args.batch_size, shuffle=False, num_workers=args.num_workers,
                                         pin_memory=device.type == "cuda")
    model, cond_stage_model, vae = load(args, device)
    print("Finish loading model")
    save_dir = os.path.join(args.out_dir, "mask2image_generated_samples", args.dataset)
    os.makedirs(save_dir, exist_ok=True)
    from PIL import Image
    for i, seg in enumerate(loader):
        u8 = synthesize(args, model, cond_stage_model, vae, seg.to(device, non_blocking=True)).cpu().numpy()
        for j, x in enumerate(u8):
            Image.fromarray(x).save(os.path.join(save_dir, "{}.jpg".format(i * args.batch_size + j)))
        print("generating batch ", i)
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
