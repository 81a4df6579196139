#!/usr/bin/env python
"""Drop-in name for the reference's inpainting CLI (downstream_tasks/test_flow_latent_inpainting.py): same flags, H100-native
execution."""
from lfm_b200.cli_inpaint import main

if __name__ == "__main__":
    raise SystemExit(main())
