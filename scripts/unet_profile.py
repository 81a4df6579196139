"""celeb512 ADM UNetModel forward, batch 32 (BASELINE.json configs[3] network) - used under ncu and for timing.

    python scripts/unet_profile.py [B] [iters] [in_channels]

in_channels > 4 times the same network concat-conditioned (the downstream tasks' WrapperCondFlow: the condition's
in_channels - 4 channels concatenated to the latents), as lfm_forward evaluates it."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import lfm_b200  # noqa: E402
from lfm_b200.synthetic import synthetic_unet_state_dict  # noqa: E402

B = int(sys.argv[1]) if len(sys.argv) > 1 else 32
iters = int(sys.argv[2]) if len(sys.argv) > 2 else 3
in_ch = int(sys.argv[3]) if len(sys.argv) > 3 else 4
dev = torch.device("cuda:0")
with torch.device("meta"):
    net = lfm_b200.UNetModel(image_size=64, in_channels=in_ch, model_channels=256, out_channels=4, num_res_blocks=2,
                             attention_resolutions=(16, 8), channel_mult=(1, 2, 2, 2, 4), num_heads=4, use_scale_shift_norm=True)
sd = synthetic_unet_state_dict(net, 1)
net = net.to_empty(device="cpu")
net.load_state_dict(sd, strict=True)
net = net.to(dev)
x = torch.randn(B, in_ch, 64, 64, device=dev)
t = torch.tensor(0.5, device=dev)
for _ in range(2):
    net(t, x)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(iters):
    v = net(t, x)
e1.record()
torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / iters
print(f"celeb512 UNet forward in_channels={in_ch} B={B}: {ms:.2f} ms/NFE, {B * 189.72e9 / ms / 1e9:.1f} TFLOP/s, launches/NFE {net.launch_count() // (iters + 2)}")
