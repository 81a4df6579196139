"""Build liblfm_b200.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU).

    python -m lfm_b200.build [--force]

The .so is a build product (git-ignored): build() of __graft_entry__.py or this module makes it.
"""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "csrc", "lfm_api.cu")
DEPS = [os.path.join(HERE, "csrc", f) for f in os.listdir(os.path.join(HERE, "csrc"))] + [
    os.path.join(os.path.dirname(HERE), "include", "lfm_b200.h")]
OUT = os.path.join(HERE, "liblfm_b200.so")


def nvcc_path():
    for p in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc")):
        if p and os.path.exists(p):
            return p
    raise RuntimeError("nvcc not found")


def needs_build():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    return any(os.path.getmtime(d) > t for d in DEPS)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return OUT
    cmd = [nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
           "-shared", "-Xcompiler", "-fPIC", "-o", OUT, SRC]
    if verbose:
        cmd.insert(-3, "-Xptxas")
        cmd.insert(-3, "-v")
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + r.stdout + r.stderr)
    if verbose:
        print(r.stderr)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
