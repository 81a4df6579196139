"""Inpainting command line (downstream_tasks/test_flow_latent_inpainting.py), running on liblfm_b200.so.

    python test_flow_latent_inpainting.py --exp inpaint_exp --dataset celeba_256 --epoch_id 500 --batch_size 50 \
        --method dopri5 --pretrained_autoencoder_ckpt ./sd-vae-ft-mse

Same flags and defaults as the reference (test_flow_latent_inpainting.py:170-224), the dataset semantics of its
``CustomizedInpaintingEvalDataset`` and its checkpoint, ``./saved_info/latent_flow_inpaint/{dataset}/{exp}/model_{epoch}.pth``
with the "module." prefix stripped.  Per batch: the masked image is encoded (``latent_dist.sample() * scale_factor``), the
mask is resized to the latents (nearest), the two make the 5-channel condition of the 9-channel UNetModel, the solver runs
``WrapperCondFlow(model, c)`` from ``z_0 ~ N(0, I)``, the result is decoded and pasted into the hole:
``fake * m + (1 - m) * image`` in [0, 1], written as ``{index}.jpg`` under ``{out_dir}/inpainting_generated_samples/{dataset}/``.
Encoder, UNet, solver and decoder all run natively.

Differences, all deliberate:
  * the paths the reference hard-codes are flags with its values as defaults: ``--gt_dir``, ``--mask_dir``, ``--num_images``
    (its dataset length), ``--out_dir``; ``--num_workers`` is its DataLoader's 4;
  * ``--synthetic_init SEED``, ``--synthetic_vae SEED`` and ``--device`` as in lfm_b200.cli;
  * the reference calls ``save_image(x, path, normalized=True)``, which raises TypeError on current torchvision (make_grid has
    no ``normalized`` argument); the files here hold what ``save_image(x, path)`` writes, ``(x * 255 + 0.5).clamp(0, 255)`` as uint8;
  * the CPU and CUDA generators are seeded with ``--seed`` (the reference seeds 42 and ignores it); ``z_0`` is drawn on the CPU
    as there, but its stream is not the reference's, which also depends on module initialisation and DataLoader worker seeding.
"""
from __future__ import annotations

import argparse
import os
import types

import numpy as np
import torch
import torch.nn.functional as F

from . import cli


def build_parser():
    p = argparse.ArgumentParser("ddgan parameters")
    p.add_argument("--seed", type=int, default=1024)
    p.add_argument("--compute_fid", action="store_true", default=False)
    p.add_argument("--epoch_id", type=int, default=500)
    p.add_argument("--image_size", type=int, default=256)
    p.add_argument("--num_in_channels", type=int, default=9)
    p.add_argument("--num_out_channels", type=int, default=4)
    p.add_argument("--nf", type=int, default=256)
    p.add_argument("--centered", action="store_false", default=True)
    p.add_argument("--resamp_with_conv", type=bool, default=True)
    p.add_argument("--num_res_blocks", type=int, default=2)
    p.add_argument("--num_heads", type=int, default=4)
    p.add_argument("--num_head_upsample", type=int, default=-1)
    p.add_argument("--num_head_channels", type=int, default=-1)
    p.add_argument("--attn_resolutions", nargs="+", type=int, default=(16, 8))
    p.add_argument("--ch_mult", nargs="+", type=int, default=(1, 2, 3, 4))
    p.add_argument("--dropout", type=float, default=0.0)
    p.add_argument("--num_classes", type=int, default=None)
    p.add_argument("--use_scale_shift_norm", type=bool, default=True)
    p.add_argument("--resblock_updown", type=bool, default=False)
    p.add_argument("--use_new_attention_order", type=bool, default=False)
    p.add_argument("--scale_factor", type=float, default=0.18215)
    p.add_argument("--exp", default="latent_kl_exp1")
    p.add_argument("--real_img_dir", default="./pytorch_fid/cifar10_train_stat.npy")
    p.add_argument("--dataset", default="celeba_256")
    p.add_argument("--num_timesteps", type=int, default=200)
    p.add_argument("--batch_size", type=int, default=50)
    p.add_argument("--atol", type=float, default=1e-5)
    p.add_argument("--rtol", type=float, default=1e-5)
    p.add_argument("--method", type=str, default="dopri5",
                   choices=["dopri5", "dopri8", "adaptive_heun", "bosh3", "euler", "midpoint", "rk4"])
    p.add_argument("--step_size", type=float, default=0.01)
    p.add_argument("--perturb", action="store_true", default=False)
    p.add_argument("--pretrained_autoencoder_ckpt", type=str, default="../stabilityai/sd-vae-ft-mse")
    # additions
    p.add_argument("--gt_dir", type=str, default="./gt_celeb/", help="ground-truth images {index:06d}.jpg")
    p.add_argument("--mask_dir", type=str, default="./dataset/masks_val_256_small_eval", help="masks {index:06d}.png")
    p.add_argument("--num_images", type=int, default=2993, help="images of the evaluation set")
    p.add_argument("--num_workers", type=int, default=4, help="DataLoader workers")
    p.add_argument("--out_dir", type=str, default=".")
    p.add_argument("--device", type=str, default=None, help="cuda:N (default: cuda:0)")
    p.add_argument("--synthetic_init", type=int, default=None, metavar="SEED", help="seeded UNet weights instead of a checkpoint")
    p.add_argument("--synthetic_vae", type=int, default=None, metavar="SEED", help="seeded VAE weights instead of a checkpoint")
    return p


class InpaintingEvalDataset(torch.utils.data.Dataset):
    """CustomizedInpaintingEvalDataset: image ``{i:06d}.jpg`` (RGB) and mask ``{i:06d}.png``; mask = 1 - png / 255 (1 marks
    the hole), masked = (1 - mask) * image; all three mapped to [-1, 1], the mask as [1, H, W]."""

    def __init__(self, indir, inmasked, length=2993):
        self.indir, self.inmasked, self.length = indir, inmasked, length

    def __len__(self):
        return self.length

    def __getitem__(self, item):
        from PIL import Image
        img = np.array(Image.open(os.path.join(self.indir, f"{item:06d}.jpg")).convert("RGB"))
        img = np.transpose(img, (2, 0, 1))
        mask = torch.from_numpy(np.array(Image.open(os.path.join(self.inmasked, f"{item:06d}.png"))))
        mask = 1 - mask / 255.0
        img = torch.from_numpy(img.astype(np.float32) / 255.0)
        masked_img = (1 - mask) * img
        return img * 2.0 - 1.0, (mask * 2.0 - 1.0).unsqueeze(0), masked_img * 2.0 - 1.0


def load(args, device):
    """The 9-channel UNetModel (get_flow_model) and the AutoencoderKL with its encoder, loaded as lfm_b200.cli loads them."""
    if args.synthetic_vae is None and not os.path.isdir(args.pretrained_autoencoder_ckpt):
        raise SystemExit(f"'{args.pretrained_autoencoder_ckpt}' is not a local diffusers directory (no hub access here): "
                         "inpainting needs the VAE encoder - pass a local copy or --synthetic_vae SEED")
    margs = types.SimpleNamespace(**vars(args), use_origin_adm=True, layout=False)
    ckpt = "./saved_info/latent_flow_inpaint/{}/{}/model_{}.pth".format(args.dataset, args.exp, args.epoch_id)
    model = cli.load_model(margs, device, ckpt_path=ckpt)
    vargs = types.SimpleNamespace(no_decode=False, vae="native", synthetic_vae=args.synthetic_vae,
                                  pretrained_autoencoder_ckpt=args.pretrained_autoencoder_ckpt)
    return model, cli.load_vae(vargs, device, with_encoder=True)


def inpaint(args, model, vae, image, mask, masked_image):
    """One batch of test_flow_latent_inpainting.py:144-170 on the device: [B, 3, H, W] images in [-1, 1] and [B, 1, H, W]
    masks -> the composited images as uint8 NHWC [B, H, W, 3] (what save_image writes)."""
    from .downstream import WrapperCondFlow, sample_from_model
    device = image.device
    c = vae.encode(masked_image).latent_dist.sample().mul_(args.scale_factor)
    cc = F.interpolate(mask, size=c.shape[-2:])
    c = torch.cat((c, cc), dim=1)
    z_0 = torch.randn(image.size(0), 4, args.image_size // 8, args.image_size // 8).to(device)
    fake_sample = sample_from_model(WrapperCondFlow(model, c), z_0, args)[-1]
    fake_image = (vae.decode(fake_sample / args.scale_factor).sample + 1.0) / 2.0
    mask, image = (mask + 1.0) / 2.0, (image + 1.0) / 2.0
    out = fake_image * mask + (1 - mask) * image
    return out.mul(255).add_(0.5).clamp_(0, 255).permute(0, 2, 3, 1).to(torch.uint8)


def main(argv=None):
    args = build_parser().parse_args(argv)
    torch.set_grad_enabled(False)
    device = torch.device(args.device if args.device else "cuda:0")
    torch.manual_seed(args.seed)
    if device.type == "cuda":
        torch.cuda.set_device(device)
        torch.cuda.manual_seed_all(args.seed)
    dataset = InpaintingEvalDataset(args.gt_dir, args.mask_dir, args.num_images)
    loader = torch.utils.data.DataLoader(dataset, batch_size=args.batch_size, shuffle=False, num_workers=args.num_workers,
                                         pin_memory=device.type == "cuda")
    model, vae = load(args, device)
    print("Finish loading model")
    save_dir = os.path.join(args.out_dir, "inpainting_generated_samples", args.dataset)
    os.makedirs(save_dir, exist_ok=True)
    from PIL import Image
    for i, (image, mask, masked_image) in enumerate(loader):
        u8 = inpaint(args, model, vae, image.to(device), mask.to(device), masked_image.to(device)).cpu().numpy()
        for j, x in enumerate(u8):
            Image.fromarray(x).save(os.path.join(save_dir, "{}.jpg".format(i * image.size(0) + j)))
        print("generating batch ", i)
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
