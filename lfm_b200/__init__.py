"""lfm_b200 - H100-native (sm_90a) latent flow-matching sampler: the sampling hot path of VinAIResearch/LFM.

Host-side mirror of the reference's interface for this path; the compute lives in liblfm_b200.so
(hand-written CUDA: wgmma GEMM, mma.sync attention, TMA, CUDA-graph solver loop) behind the C ABI in
include/lfm_b200.h.  Importing this package never touches the GPU; calling into it without the built library
or without an H100 raises - there is no CPU or eager-PyTorch fallback.
"""
from .network import DiT, DiT_models, create_network, get_flow_model  # noqa: F401
from .unet import UNetModel  # noqa: F401
from .edm import DhariwalUNet, get_edm_network  # noqa: F401
from .vae import AutoencoderKL, synthetic_vae_state_dict  # noqa: F401
from .solvers import (ADAPTIVE_SOLVER, FIXER_SOLVER, euler_time_grid, karras_sample, sample_from_model,  # noqa: F401
                      sample_from_model_with_fixed_step_solve, sample_from_model_with_fixed_step_solver)

__all__ = ["DiT", "UNetModel", "DhariwalUNet", "AutoencoderKL", "get_edm_network", "DiT_models", "create_network", "get_flow_model", "karras_sample", "sample_from_model",
           "sample_from_model_with_fixed_step_solver", "euler_time_grid"]
