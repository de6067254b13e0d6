#!/usr/bin/env python
"""Packages the UNMODIFIED reference implementation of the hot path so that it can run where the checkout is absent.

    python oracle/make_ref.py            # -> oracle/_ref/trainer_ref.zip  (git-ignored; build() runs it too)

The reference is pure Python (no native code, nothing to compile): its `trainer` package is zipped from the layout-dm
checkout (REF_PKG_PARENT below) -- no source file is copied into the repository tree or its history -- and imported
from the archive (zipimport) together with the import stand-ins of oracle/ref_shims (hydra / omegaconf / torch_geometric
... are not installed in this image; none of them is on the arithmetic path of `LayoutDM.sample()`, SURVEY.md 8c).
Consumers: `bench.py --impl reference` / `gpu_eager_baseline` (the reference's own `LayoutDM.sample`, layoutdm.py:77-88,
timed on the host cores / eagerly on the GPU) and the drop-in test of `patch_reference_model`.  TEST / BENCH
INFRASTRUCTURE ONLY: nothing under layoutdm_b200/ imports it.
"""
from __future__ import annotations

import os
import sys
import zipfile

HERE = os.path.dirname(os.path.abspath(__file__))
REF_PKG_PARENT = "/root/reference/src/trainer"          # the read-only reference checkout
OUT_DIR = os.path.join(HERE, "_ref")
OUT = os.path.join(OUT_DIR, "trainer_ref.zip")


def build(force: bool = False) -> str | None:
    """returns the archive path, or None when the reference checkout is absent and no archive was packaged before"""
    src = os.path.join(REF_PKG_PARENT, "trainer")
    if not os.path.isdir(src):
        return OUT if os.path.exists(OUT) else None
    files = []
    for root, _, names in os.walk(src):
        for n in sorted(names):
            if n.endswith(".py"):
                files.append(os.path.join(root, n))
    files.sort()
    newest = max(os.path.getmtime(f) for f in files)
    if not force and os.path.exists(OUT) and os.path.getmtime(OUT) >= newest:
        return OUT
    os.makedirs(OUT_DIR, exist_ok=True)
    tmp = OUT + ".tmp"
    with zipfile.ZipFile(tmp, "w", zipfile.ZIP_DEFLATED) as z:
        for f in files:
            z.write(f, os.path.relpath(f, REF_PKG_PARENT))
    os.replace(tmp, OUT)
    return OUT


if __name__ == "__main__":
    p = build(force="--force" in sys.argv)
    print(p if p else "reference not available and no prebuilt archive")
