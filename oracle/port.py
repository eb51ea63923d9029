"""TEST INFRASTRUCTURE — ctypes handle on the plain-C restatement (oracle/s2o_*.c -> oracle/libs2oracle.so).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may import this module; the product never does.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from solver2d_b200 import device

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "libs2oracle.so")


def build(force: bool = False) -> str:
    srcs = [os.path.join(HERE, f) for f in os.listdir(HERE) if f.startswith("s2o_") and f.endswith((".c", ".inc"))]
    if force or not os.path.exists(SO) or any(os.path.getmtime(s) > os.path.getmtime(SO) for s in srcs):
        subprocess.run(["make", "-C", HERE, "oracle"], check=True, capture_output=True)
    return SO


class Oracle:
    def __init__(self, path: str | None = None):
        """`path`: a library built from oracle/s2o_solver.c (default: oracle/libs2oracle.so, built on demand)."""
        self.lib = C.CDLL(build() if path is None else path)
        args = [C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int,
                C.POINTER(device.StepContext), C.c_float, C.c_float]
        self.lib.s2o_solve.restype = C.c_int
        self.lib.s2o_solve.argtypes = args
        self.lib.s2o_solve_dp.restype = C.c_int
        self.lib.s2o_solve_dp.argtypes = args + [C.c_void_p]

    def solve(self, solver_type: int, bodies: np.ndarray, contacts: np.ndarray, joints: np.ndarray, ctx: device.StepContext,
              order: np.ndarray | None = None, gravity=(0.0, -10.0), dp: np.ndarray | None = None):
        """Runs the restated solver stage in place on copies of the rows and returns (bodies, contacts, joints).
        `order`: optional visiting order, entries >= 0 = contact row, < 0 = joint slot (-1 - k).
        `dp`: optional (len(bodies), 2) delta positions the bodies start the stage with (zero if not given); when given,
        the delta positions the stage leaves are returned as a fourth item."""
        bodies = np.ascontiguousarray(bodies.copy(), dtype=device.BODY_ROW)
        contacts = np.ascontiguousarray(contacts.copy(), dtype=device.CONTACT_ROW)
        joints = np.ascontiguousarray(joints.copy(), dtype=device.JOINT_ROW)
        if order is not None:
            order = np.ascontiguousarray(order, dtype=np.int32)
        args = (solver_type, bodies.ctypes.data, len(bodies), contacts.ctypes.data, len(contacts), joints.ctypes.data,
                len(joints), None if order is None else order.ctypes.data, 0 if order is None else len(order), C.byref(ctx),
                gravity[0], gravity[1])
        if dp is None:
            rc = self.lib.s2o_solve(*args)
        else:
            dp = np.array(dp, dtype=np.float32, order="C", copy=True)
            assert dp.shape == (len(bodies), 2), dp.shape
            rc = self.lib.s2o_solve_dp(*args, dp.ctypes.data)
        if rc != 0:
            raise NotImplementedError(f"oracle: solver type {solver_type} not restated")
        return (bodies, contacts, joints) if dp is None else (bodies, contacts, joints, dp)


_cached = None


def load() -> Oracle:
    global _cached
    if _cached is None:
        _cached = Oracle()
    return _cached
