"""The joint oracle (tests/joint_oracle.c): oracle/s2o_solver.c with every joint type the reference lacks.

Compiled on first use with the oracle's own flags into a per-user temporary directory (the repository tree stays
untouched), keyed by the hash of every source it includes. `solve` has the signature of oracle.port.Oracle.solve.
"""
from __future__ import annotations

import glob
import hashlib
import os
import subprocess
import tempfile

from helpers import ROOT
from oracle import port

SRC = os.path.join(ROOT, "tests", "joint_oracle.c")


def _sources() -> list[str]:
    return [SRC] + sorted(glob.glob(os.path.join(ROOT, "tests", "joint_oracle", "*.inc"))) \
        + [os.path.join(ROOT, "solver2d_b200", "csrc", "shared", f) for f in ("s2_collide.h", "s2_distance_joint.h", "s2_gear_joint.h")] \
        + sorted(glob.glob(os.path.join(ROOT, "oracle", "s2o_*"))) \
        + sorted(glob.glob(os.path.join(ROOT, "include", "**", "*.h"), recursive=True))


def build() -> str:
    h = hashlib.sha1()
    for f in _sources():
        with open(f, "rb") as fh:
            h.update(fh.read())
    out_dir = os.path.join(tempfile.gettempdir(), f"s2o_joint_{os.getuid()}")
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, f"libs2oracle_joint_{h.hexdigest()[:16]}.so")
    if not os.path.exists(so):
        tmp = f"{so}.{os.getpid()}.tmp"
        subprocess.run(["gcc", "-std=gnu17", "-O2", "-fPIC", "-fvisibility=default", "-Wall", "-I" + os.path.join(ROOT, "include"),
                        "-shared", "-o", tmp, SRC, "-lm"], check=True, capture_output=True)
        os.replace(tmp, so)
    return so


_cached = None


def load() -> port.Oracle:
    global _cached
    if _cached is None:
        _cached = port.Oracle(build())
    return _cached
