"""The gear joint's oracle (tests/gear_oracle.c): the pulley oracle with gear rows.

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

SRC = os.path.join(ROOT, "tests", "gear_oracle.c")


def _sources() -> list[str]:
    return [SRC] + [os.path.join(ROOT, "tests", f"{name}_oracle.c") for name in ("pulley", "wheel", "distance", "spring", "prismatic")] \
        + [os.path.join(ROOT, "solver2d_b200", "csrc", "shared", f) for f in ("s2_collide.h", "s2_distance_joint.h", "s2_gear_joint.h")] \
        + sorted(glob.glob(os.path.join(ROOT, "oracle", "s2o_*"))) \
        + sorted(glob.glob(os.path.join(ROOT, "include", "**", "*.h"), recursive=True))


def build() -> str:
    h = hashlib.sha1()
    for f in _sources():
        with open(f, "rb") as fh:
            h.update(fh.read())
    out_dir = os.path.join(tempfile.gettempdir(), f"s2o_gear_{os.getuid()}")
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, f"libs2oracle_gear_{h.hexdigest()[:16]}.so")
    if not os.path.exists(so):
        tmp = f"{so}.{os.getpid()}.tmp"
        subprocess.run(["gcc", "-std=gnu17", "-O2", "-fPIC", "-fvisibility=default", "-Wall", "-I" + os.path.join(ROOT, "include"),
                        "-shared", "-o", tmp, SRC, "-lm"], check=True, capture_output=True)
        os.replace(tmp, so)
    return so


class GearOracle(port.Oracle):
    def __init__(self):  # noqa: D107 - the same entry points as the oracle's, from the gear build
        super().__init__(build())


_cached = None


def load() -> GearOracle:
    global _cached
    if _cached is None:
        _cached = GearOracle()
    return _cached
