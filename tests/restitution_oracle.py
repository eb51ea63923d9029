"""Restitution (DESIGN.md §3.7) restated in float32 numpy on top of the plain-C oracle of the solver stage.

solve() = capture from the input rows, the variant's whole stage in the oracle (restitution off: oracle/port.py's solve),
then the restitution pass in the visiting order. Every float operation is the device's, one by one, in the same order
(include/solver2d/math.h inlines, no fused multiply-add), so the result is bit-exact against the device."""
from __future__ import annotations

import numpy as np

from solver2d_b200 import capi

f32 = np.float32
XPBD = capi.SOLVER["XPBD"]


def capture(bodies: np.ndarray, contacts: np.ndarray) -> dict:
    """Per contact row and point, at the stage-start state: approach speed vr, normal mass, anchors rA, rB."""
    A = bodies[contacts["bodyA"]]
    B = bodies[contacts["bodyB"]]
    nx, ny = contacts["normal"][:, 0], contacts["normal"][:, 1]
    mA, mB, iA, iB = A["invMass"], B["invMass"], A["invI"], B["invI"]
    sA, cA, sB, cB = A["rot"][:, 0], A["rot"][:, 1], B["rot"][:, 0], B["rot"][:, 1]
    vAx, vAy, wA = A["linearVelocity"][:, 0], A["linearVelocity"][:, 1], A["angularVelocity"]
    vBx, vBy, wB = B["linearVelocity"][:, 0], B["linearVelocity"][:, 1], B["angularVelocity"]
    out = {"vr": [], "mN": [], "rA": [], "rB": []}
    for j in range(2):
        p = contacts["points"][:, j]
        lAx = p["localAnchorA"][:, 0] - A["localCenter"][:, 0]
        lAy = p["localAnchorA"][:, 1] - A["localCenter"][:, 1]
        lBx = p["localAnchorB"][:, 0] - B["localCenter"][:, 0]
        lBy = p["localAnchorB"][:, 1] - B["localCenter"][:, 1]
        rAx, rAy = cA * lAx - sA * lAy, sA * lAx + cA * lAy  # s2RotateVector
        rBx, rBy = cB * lBx - sB * lBy, sB * lBx + cB * lBy
        dx = (vBx + (-wB) * rBy) - (vAx + (-wA) * rAy)  # s2CrossSV(w, r) = {-w r.y, w r.x}
        dy = (vBy + wB * rBx) - (vAy + wA * rAx)
        vr = nx * dx + ny * dy
        rnA = rAx * ny - rAy * nx
        rnB = rBx * ny - rBy * nx
        k = mA + mB + iA * rnA * rnA + iB * rnB * rnB
        with np.errstate(divide="ignore"):
            mN = np.where(k > f32(0), f32(1) / k, f32(0)).astype(f32)
        out["vr"].append(vr.astype(f32))
        out["mN"].append(mN)
        out["rA"].append(np.stack([rAx, rAy], 1).astype(f32))
        out["rB"].append(np.stack([rBx, rBy], 1).astype(f32))
    return out


def restitution_pass(bodies: np.ndarray, contacts: np.ndarray, cap: dict, items, threshold: float) -> int:
    """Gauss-Seidel over the contacts of `items` (entries >= 0 = contact row; joints < 0 are skipped) in order, in place.
    Returns the number of points that bounced."""
    thr = f32(threshold)
    e_all = contacts["restitution"]
    count = contacts["pointCount"]
    lam0 = contacts["points"]["normalImpulse"]
    # which points apply is known up front: a point's stored impulse only changes when the pass visits that very point
    hit = np.zeros((len(contacts), 2), dtype=bool)
    for j in range(2):
        hit[:, j] = (e_all != 0) & (count > j) & ~(cap["vr"][j] > -thr) & (lam0[:, j] != 0)
    rows = set(np.nonzero(hit.any(axis=1))[0].tolist())
    bounced = 0
    for slot in (int(t) for t in items if t >= 0 and int(t) in rows):
        a, b = int(contacts["bodyA"][slot]), int(contacts["bodyB"][slot])
        e = f32(e_all[slot])
        nx, ny = f32(contacts["normal"][slot, 0]), f32(contacts["normal"][slot, 1])
        mA, mB = f32(bodies["invMass"][a]), f32(bodies["invMass"][b])
        iA, iB = f32(bodies["invI"][a]), f32(bodies["invI"][b])
        vAx, vAy = (f32(x) for x in bodies["linearVelocity"][a])
        vBx, vBy = (f32(x) for x in bodies["linearVelocity"][b])
        wA, wB = f32(bodies["angularVelocity"][a]), f32(bodies["angularVelocity"][b])
        for j in range(2):
            if not hit[slot, j]:
                continue
            lam = f32(contacts["points"]["normalImpulse"][slot, j])
            rAx, rAy = (f32(x) for x in cap["rA"][j][slot])
            rBx, rBy = (f32(x) for x in cap["rB"][j][slot])
            dx = (vBx + (-wB) * rBy) - (vAx + (-wA) * rAy)
            dy = (vBy + wB * rBx) - (vAy + wA * rAx)
            vn = dx * nx + dy * ny
            impulse = -f32(cap["mN"][j][slot]) * (vn + e * f32(cap["vr"][j][slot]))
            new = lam + impulse
            new = new if new > f32(0) else f32(0)
            impulse = new - lam
            contacts["points"]["normalImpulse"][slot, j] = new
            Px, Py = impulse * nx, impulse * ny
            vAx, vAy = vAx - mA * Px, vAy - mA * Py
            wA = wA - iA * (rAx * Py - rAy * Px)
            vBx, vBy = vBx + mB * Px, vBy + mB * Py
            wB = wB + iB * (rBx * Py - rBy * Px)
            bounced += 1
        if mA != 0 or iA != 0:
            bodies["linearVelocity"][a] = (vAx, vAy)
            bodies["angularVelocity"][a] = wA
        if mB != 0 or iB != 0:
            bodies["linearVelocity"][b] = (vBx, vBy)
            bodies["angularVelocity"][b] = wB
    return bounced


def solve(O, solver_type: int, bodies, contacts, joints, ctx, order=None, gravity=(0.0, -10.0), threshold: float = 1.0):
    """The solver stage with restitution on: (bodies, contacts, joints, points that bounced)."""
    cap = capture(bodies, contacts)
    ob, oc, oj = O.solve(solver_type, bodies, contacts, joints, ctx, order=order, gravity=gravity)
    if ctx.dt == 0.0 or (solver_type == XPBD and ctx.iterations == 0):
        return ob, oc, oj, 0  # no stage (s2Solve_XPBD returns early) or no pass
    items = order if order is not None else np.arange(len(contacts))
    n = restitution_pass(ob, oc, cap, items, threshold)
    return ob, oc, oj, n
