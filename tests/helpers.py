"""Shared test plumbing: reference taps -> device rows, state comparison."""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ref as refmod  # noqa: E402
from solver2d_b200 import capi, device  # noqa: E402


def has_gpu() -> bool:
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def body_rows_from_ref(bf: np.ndarray, bi: np.ndarray) -> np.ndarray:
    """All body slots of a reference world as device rows (free slots are uploaded as invalid rows)."""
    F = refmod.BODY_F
    n = bf.shape[0]
    rows = np.zeros(n, dtype=device.BODY_ROW)
    rows["index"] = np.arange(n)
    rows["flags"] = np.where(bi[:, 0] == 1, device.ROW_VALID | (bi[:, 1] << 1), 0)
    rows["origin"] = bf[:, F["origin"]:F["origin"] + 2]
    rows["position"] = bf[:, F["position"]:F["position"] + 2]
    rows["rot"] = bf[:, F["rot"]:F["rot"] + 2]
    rows["linearVelocity"] = bf[:, F["v"]:F["v"] + 2]
    rows["angularVelocity"] = bf[:, F["w"]]
    rows["localCenter"] = bf[:, F["localCenter"]:F["localCenter"] + 2]
    rows["mass"] = bf[:, F["mass"]]
    rows["invMass"] = bf[:, F["invMass"]]
    rows["I"] = bf[:, F["I"]]
    rows["invI"] = bf[:, F["invI"]]
    rows["force"] = bf[:, F["force"]:F["force"] + 2]
    rows["torque"] = bf[:, F["torque"]]
    rows["linearDamping"] = bf[:, F["linearDamping"]]
    rows["angularDamping"] = bf[:, F["angularDamping"]]
    rows["gravityScale"] = bf[:, F["gravityScale"]]
    return rows


def contact_rows_from_ref(cf: np.ndarray, ci: np.ndarray):
    """Live contacts of a reference world, in pool-slot order (= the reference's Gauss-Seidel order), as device rows.
    Returns (rows, slots) where slots[i] is the reference pool slot of row i."""
    I = refmod.CONTACT_I
    slots = np.nonzero(ci[:, I["valid"]] == 1)[0]
    rows = np.zeros(len(slots), dtype=device.CONTACT_ROW)
    c = ci[slots]
    f = cf[slots]
    rows["shapeA"] = c[:, I["shapeA"]]
    rows["shapeB"] = c[:, I["shapeB"]]
    rows["bodyA"] = c[:, I["bodyA"]]
    rows["bodyB"] = c[:, I["bodyB"]]
    rows["pointCount"] = c[:, I["pointCount"]]
    rows["frictionPersisted"] = c[:, I["frictionPersisted"]]
    rows["friction"] = f[:, 0]
    rows["normal"] = f[:, 1:3]
    rows["cacheMetric"] = f[:, 3]
    rows["cacheCount"] = c[:, I["cacheCount"]]
    for k in range(3):
        rows["cacheIndexA"][:, k] = (c[:, I["cacheA"]] >> (8 * k)) & 0xFF
        rows["cacheIndexB"][:, k] = (c[:, I["cacheB"]] >> (8 * k)) & 0xFF
    P = refmod.POINT_F
    for j in range(2):
        base = refmod.CONTACT_F["points"] + refmod.POINT_STRIDE * j
        q = f[:, base:base + refmod.POINT_STRIDE]
        pt = rows["points"][:, j]
        for name in ("localAnchorA", "localAnchorB", "frictionAnchorA", "frictionAnchorB", "frictionNormalA",
                     "frictionNormalB"):
            pt[name] = q[:, P[name]:P[name] + 2]
        pt["separation"] = q[:, P["separation"]]
        pt["normalImpulse"] = q[:, P["normalImpulse"]]
        pt["tangentImpulse"] = q[:, P["tangentImpulse"]]
        pt["id"] = c[:, I["id0"] + j]
        pt["persisted"] = c[:, I["persisted0"] + j]
        rows["points"][:, j] = pt
    return rows, slots


STICKY_FIELDS = ("frictionAnchorA", "frictionAnchorB", "frictionNormalA", "frictionNormalB")


def carry_sticky_friction(rows, keys, solved):
    """The friction anchors and normals a TGS_Sticky solve writes into the manifolds (reference
    src/solve_tgs_sticky.c:147-163) are carried into the next step's manifolds by s2UpdateContact: a new point takes those
    of the FIRST old point with its id, an unmatched point starts at zero (reference src/contact.c:317-358). The reference
    world is advanced with the oracle's impulses only, so this restates that carry-over on its post-collide rows, from the
    oracle's rows of the previous step. Which points matched is checked against the reference's own persisted flags."""
    for k, key in enumerate(keys.tolist()):
        old = solved.get(key)
        for i in range(2):
            j = -1
            if old is not None and i < rows["pointCount"][k]:
                j = next((j for j in range(old["pointCount"]) if old["points"]["id"][j] == rows["points"]["id"][k, i]), -1)
            if i < rows["pointCount"][k]:
                assert (j >= 0) == bool(rows["points"]["persisted"][k, i]), "id matching differs from the reference's"
            for name in STICKY_FIELDS:
                rows["points"][name][k, i] = old["points"][name][j] if j >= 0 else 0.0


def joint_rows_from_ref(jf: np.ndarray, ji: np.ndarray) -> np.ndarray:
    I, F = refmod.JOINT_I, refmod.JOINT_F
    n = jf.shape[0]
    rows = np.zeros(n, dtype=device.JOINT_ROW)
    rows["index"] = np.arange(n)
    valid = ji[:, I["valid"]] == 1
    flags = np.where(valid, device.ROW_VALID | (ji[:, I["type"]] << 1), 0)
    flags |= np.where(valid & (ji[:, I["enableLimit"]] == 1), device.JOINT_ENABLE_LIMIT, 0)
    flags |= np.where(valid & (ji[:, I["enableMotor"]] == 1), device.JOINT_ENABLE_MOTOR, 0)
    flags |= np.where(valid & (ji[:, I["collideConnected"]] == 1), device.JOINT_COLLIDE_CONNECTED, 0)
    rows["flags"] = flags
    rows["bodyA"] = ji[:, I["bodyA"]]
    rows["bodyB"] = ji[:, I["bodyB"]]
    rows["localOriginAnchorA"] = jf[:, 0:2]
    rows["localOriginAnchorB"] = jf[:, 2:4]
    rows["impulse"] = jf[:, 4:6]
    rows["motorImpulse"] = jf[:, F["motorImpulse"]]
    rows["lowerImpulse"] = jf[:, F["lowerImpulse"]]
    rows["upperImpulse"] = jf[:, F["upperImpulse"]]
    rows["maxMotorTorque"] = jf[:, F["maxMotorTorque"]]
    rows["motorSpeed"] = jf[:, F["motorSpeed"]]
    rows["referenceAngle"] = jf[:, F["referenceAngle"]]
    rows["lowerAngle"] = jf[:, F["lowerAngle"]]
    rows["upperAngle"] = jf[:, F["upperAngle"]]
    rows["hertz"] = jf[:, F["hertz"]]
    rows["dampingRatio"] = jf[:, F["dampingRatio"]]
    rows["target"] = jf[:, F["target"]:F["target"] + 2]
    return rows


def load_device_world_from_ref(dev: device.Device, R: refmod.Reference, wid, solver: str) -> device.DeviceWorld:
    """Mirror the current state of a reference world (bodies, joints, contacts in pool order) into a device world."""
    dw = dev.create_world(capi.SOLVER[solver])
    bf, bi = R.bodies(wid)
    dw.upload_bodies(body_rows_from_ref(bf, bi), bf.shape[0])
    jf, ji = R.joints(wid)
    dw.upload_joints(joint_rows_from_ref(jf, ji), jf.shape[0])
    cf, ci = R.contacts(wid)
    rows, slots = contact_rows_from_ref(cf, ci)
    dw.upload_contacts(rows)
    dw.ref_contact_slots = slots
    return dw


def compare_bodies(dev_rows: np.ndarray, bf: np.ndarray, bi: np.ndarray) -> dict:
    """Max abs differences between downloaded device body rows and a reference body dump (valid slots only)."""
    F = refmod.BODY_F
    valid = bi[:, 0] == 1
    d = {}
    d["pos"] = float(np.abs(dev_rows["position"][valid] - bf[valid, F["position"]:F["position"] + 2]).max())
    d["rot"] = float(np.abs(dev_rows["rot"][valid] - bf[valid, F["rot"]:F["rot"] + 2]).max())
    d["v"] = float(np.abs(dev_rows["linearVelocity"][valid] - bf[valid, F["v"]:F["v"] + 2]).max())
    d["w"] = float(np.abs(dev_rows["angularVelocity"][valid] - bf[valid, F["w"]]).max())
    d["origin"] = float(np.abs(dev_rows["origin"][valid] - bf[valid, F["origin"]:F["origin"] + 2]).max())
    return d


def bit_equal(a: np.ndarray, b: np.ndarray) -> bool:
    a = np.ascontiguousarray(a, dtype=np.float32)
    b = np.ascontiguousarray(b, dtype=np.float32)
    return bool(np.array_equal(a.view(np.uint32), b.view(np.uint32)))
