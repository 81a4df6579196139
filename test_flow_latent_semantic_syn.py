#!/usr/bin/env python
"""Drop-in name for the reference's semantic-synthesis CLI (downstream_tasks/test_flow_latent_semantic_syn.py): same flags,
H100-native execution."""
from lfm_b200.cli_semantic import main

if __name__ == "__main__":
    raise SystemExit(main())
