"""Reference-equivalent EAGER PyTorch on the GPU (test tooling; uses the oracle restatement, which is the reference's
algorithm op for op): DiT-L/2 forward, batch 64, fp32 with TF32 off (test_flow_latent.py:103 leaves TF32 commented
out), TF32 on (test_flow_latent_ddp.py:23) and bf16 autocast.  Prints NFE*img/s and Euler-50 images/s."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import dit as odit  # noqa: E402

dev = torch.device("cuda:0")
torch.set_default_device(dev)   # the oracle builds its small index tensors on the default device
cfg = odit.make_config("DiT-L/2", num_classes=1, label_dropout=0.0)
with torch.device("cpu"):
    sd = odit.synthetic_state_dict(cfg, 1)
sd = {k: v.to(dev) for k, v in sd.items()}
B = 64
x = torch.randn(B, 4, 32, 32, device=dev)
t = torch.tensor(0.5, device=dev)


def run(label, setup, autocast=False):
    setup()
    def f():
        if autocast:
            with torch.autocast("cuda", dtype=torch.bfloat16):
                return odit.dit_forward(sd, cfg, t, x)
        return odit.dit_forward(sd, cfg, t, x)
    for _ in range(2):
        f()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    n = 5
    for _ in range(n):
        f()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / n
    print(json.dumps({"eager_torch": label, "ms_per_nfe": round(ms, 3), "nfe_img_per_s": round(B / ms * 1e3, 1),
                      "euler50_images_per_s": round(B / ms * 1e3 / 50, 2), "tflops": round(B * 161.386856448e9 / ms / 1e9, 1)}))


def tf32(on):
    def s():
        torch.backends.cuda.matmul.allow_tf32 = on
        torch.backends.cudnn.allow_tf32 = on
    return s


run("fp32, TF32 off (test_flow_latent.py)", tf32(False))
run("fp32, TF32 on (test_flow_latent_ddp.py:23)", tf32(True))
run("bf16 autocast", tf32(True), autocast=True)
