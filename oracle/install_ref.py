"""Install the UNMODIFIED reference (a checkout of lucidrains/egnn-pytorch: EGNN_REFERENCE_SRC, else a directory
named `reference` next to this repository) into oracle/_ref.  `__graft_entry__.build()` runs it when a checkout is
found; by hand:

    [EGNN_REFERENCE_SRC=<checkout>] python oracle/install_ref.py [--force]

oracle/_ref is git-ignored and is a build product: it goes wherever the built tree goes.  When present, `bench.py --impl reference` (the reference's own torch forward on
the host cores) and the `gpu_eager_baseline` leg of `bench.py` (the reference's own PyTorch-eager forward on
the same GPU) import it; without it they fall back to oracle/egnn_torch_port.py or report it unavailable.
Nothing of the product imports it.

Recipe: the checkout may be read-only and its setup.py asks for
`setup_requires=['pytest-runner']`, which cannot be resolved offline, so the tree is copied to a
temporary directory, that one stanza is dropped from the COPY's setup.py (package files are byte
identical -- checked below by sha256), and
    pip install --no-index --no-build-isolation --no-deps --target oracle/_ref <copy>
`--no-deps` because `numba` (an install_requires of the PyG-only code path, never imported by
egnn_pytorch.py) is not needed.
"""
from __future__ import annotations

import hashlib
import os
import re
import shutil
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
TARGET = os.path.join(HERE, "_ref")
SRC = os.environ.get("EGNN_REFERENCE_SRC") or os.path.join(os.path.dirname(HERE), "..", "reference")


def _sha(path):
    return hashlib.sha256(open(path, "rb").read()).hexdigest()


def installed():
    return os.path.exists(os.path.join(TARGET, "egnn_pytorch", "egnn_pytorch.py"))


def install(force=False, quiet=True):
    """Returns 'present' | 'installed' | 'no-source'.  Raises on a failed install."""
    if installed() and not force:
        return "present"
    if not os.path.isdir(os.path.join(SRC, "egnn_pytorch")):
        return "no-source"
    tmp = tempfile.mkdtemp(prefix="egnn_ref_")
    try:
        copy = os.path.join(tmp, "src")
        shutil.copytree(SRC, copy, ignore=shutil.ignore_patterns(".git", "__pycache__"))
        sp = os.path.join(copy, "setup.py")
        txt = open(sp).read()
        txt = re.sub(r"\n\s*setup_requires\s*=\s*\[.*?\],", "", txt, flags=re.S)
        open(sp, "w").write(txt)
        if os.path.isdir(TARGET):
            shutil.rmtree(TARGET)
        cmd = [sys.executable, "-m", "pip", "install", "--no-index", "--no-build-isolation", "--no-deps",
               "--target", TARGET, copy]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError("pip install of the reference failed:\n" + res.stdout[-2000:] + res.stderr[-2000:])
        for name in os.listdir(os.path.join(SRC, "egnn_pytorch")):
            if name.endswith(".py"):
                a, b = os.path.join(SRC, "egnn_pytorch", name), os.path.join(TARGET, "egnn_pytorch", name)
                if _sha(a) != _sha(b):
                    raise RuntimeError(f"installed {name} differs from the reference source")
        if not quiet:
            print(res.stdout[-500:])
        return "installed"
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    print(install(force="--force" in sys.argv, quiet=False), TARGET)
