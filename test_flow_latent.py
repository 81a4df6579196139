#!/usr/bin/env python
"""Drop-in name for the reference's sampling CLI (test_flow_latent.py): same flags, H100-native execution."""
from lfm_b200.cli import main

if __name__ == "__main__":
    raise SystemExit(main())
