"""Scenes of tests/test_hub_capacity_gpu.py and the sizes each one is built to reach, shared with the CPU companion
tests/test_hub_capacity_cpu.py (which checks every size on the reference's own tables, without a GPU).

A hub is a movable body with more than HEAVY_DEGREE incident constraints. Its incidence list holds every live constraint
(a contact with points, a joint; a mouse joint counts on its body B only) that can move it. The sizes below are the
quantities the device decides its paths on:

* the serial overflow group's contacts, joints and distinct bodies (movable or not, as s2bOverflowBodiesKernel counts
  them), against S2B_OV_MAX_CONTACTS / _JOINTS / _BODIES (persistent.cuh);
* each body's incidence-list length, against the per-thread sorts (<= 8, 9-24), the shared-memory bitonic sort (25-2048)
  and the heap sort beyond it (solver.cu), and against HEAVY_DEGREE (warm_gather.cuh);
* the number of hubs, against the persistent grid (blocks loop over hubs);
* the colours of a hub's constraints, against S2B_MAX_COLORS.
"""
from __future__ import annotations

import numpy as np

from helpers import body_rows_from_ref, contact_rows_from_ref, joint_rows_from_ref
from solver2d_b200 import device, scenes

DT = 1.0 / 60.0
HEAVY_DEGREE = 48          # S2B_HEAVY_DEGREE: hub bodies of the regions and the block-wide warm-start gather
HUB_DEGREE = 48            # default colouring threshold (S2B_HUB_DEGREE)
OV_MAX_BODIES, OV_MAX_CONTACTS, OV_MAX_JOINTS = 1024, 2048, 256
LONG_LIST, LONG_LIST_SHARED = 24, 2048
MAX_COLORS = 64


def beam(pendulums, limits_motor=False):
    return lambda L, solver: scenes.hub_beam(L, solver, pendulums=pendulums, limits_motor=limits_motor)


def trays(trays=(), on_ground=()):
    return lambda L, solver: scenes.hub_trays(L, solver, trays=trays, on_ground=on_ground)


# name -> (builder, sizes). Sizes: "serial" = (contacts, joints, distinct bodies) of the serial group at the default
# colouring threshold; "hubs" = sorted incidence-list lengths of the bodies above HEAVY_DEGREE; "lists" = a few more
# list lengths that must occur (a multiset, checked by count).
SCENES = {
    # ---- serial group at the staging limits (1 tray + its lane + riders; riders touch nothing else)
    "bodies_1024": (trays([[1] * 1022]), dict(serial=(1023, 0, 1024), hubs=[1023])),
    "bodies_1025": (trays([[1] * 1023]), dict(serial=(1024, 0, 1025), hubs=[1024])),
    "contacts_2048": (trays([[3] * 682 + [1]]), dict(serial=(2048, 0, 685), hubs=[2048])),
    "contacts_2049": (trays([[3] * 682 + [2]]), dict(serial=(2049, 0, 685), hubs=[2049])),
    # beam: pendulums + 2 hangers + 1 mouse joint; bodies: beam, bobs, the anchor (also the mouse joint's body A)
    "joints_256": (beam(253), dict(serial=(0, 256, 255), hubs=[256])),
    "joints_257": (beam(254), dict(serial=(0, 257, 256), hubs=[257])),
    "joints_256_limits_motor": (beam(253, True), dict(serial=(0, 256, 255), hubs=[256])),
    "joints_257_limits_motor": (beam(254, True), dict(serial=(0, 257, 256), hubs=[257])),
    # ---- incidence-list lengths on either side of every sort path: 25 / 33 (bitonic, padded to 32 / 64), 512 / 513 /
    # 1025 (padded to 512 / 1024 / 2048), 3000 (heap sort); compound riders of 9-24 shapes (insertion sort), 24 and 25
    "lists": (trays([[1] * 511, [1] * 512, [9, 12, 24, 25, 33, 16] + [1] * 905, [3] * 999 + [2]], on_ground=[24, 25, 33, 8, 9]),
              dict(hubs=[512, 513, 1025, 3000], lists=[9, 9, 12, 16, 24, 24, 25, 25, 33, 33, 8])),
    # ---- more hubs than 4 x the SM count: the persistent grid (at most 4 blocks of 512 threads per SM) loops over them
    "many_hubs": (trays(on_ground=[49] * 540), dict(hubs=[49] * 540)),
    # ---- colour limit: S2B_HUB_DEGREE=0 colours a tray of 100 constraints; 64 colours, 36 overflow
    "colour_limit": (trays([[1] * 99], on_ground=[3]), dict(hubs=[100], lists=[3])),
    # ---- thresholds: degree 60 and 20 (S2B_HUB_DEGREE=100), 40 and 20 (S2B_HUB_DEGREE=30), 48 and 49 (defaults)
    "degree_60": (trays(on_ground=[60, 20]), dict(hubs=[60], lists=[20])),
    "degree_40": (trays(on_ground=[40, 20]), dict(hubs=[], lists=[40, 20])),
    "degree_48_49": (trays(on_ground=[48, 49, 2]), dict(hubs=[49], lists=[48, 2])),
}


def build_rows(R, name, solver, settle=0):
    """Reference scene `name` built for `solver`, stepped `settle` times, then collided: (bodies, contacts, joints, scene)
    rows as the device takes them. The scenes are built at rest with every contact touching, so the first collide already
    has every manifold; a step of Jacobi would knock riders off their tray. The scene is destroyed; its pile ids are
    returned in the scene object."""
    builder, _ = SCENES[name]
    sc = builder(R, solver)
    for _ in range(settle):
        sc.step(DT, 4, 2, True)
    R.step_collide(sc.world)
    bodies = body_rows_from_ref(*R.bodies(sc.world))
    contacts, _ = contact_rows_from_ref(*R.contacts(sc.world))
    joints = joint_rows_from_ref(*R.joints(sc.world))
    sc.destroy()
    return bodies, contacts, joints, sc


def movable(bodies):
    return (bodies["invMass"] != 0) | (bodies["invI"] != 0)


def item_ends(bodies, contacts, joints):
    """(ends_a, ends_b, raw_a, raw_b) of every live item, joints first (live slots in slot order), then live contacts:
    the movable endpoint or -1 (what the incidence lists hold), and the raw body index (what the serial group's body
    count takes)."""
    mov = movable(bodies)
    jl = (joints["flags"] & 1) == 1
    cl = contacts["pointCount"] > 0
    ja, jb = joints["bodyA"][jl].astype(np.int64), joints["bodyB"][jl].astype(np.int64)
    mouse = ((joints["flags"][jl] >> 1) & 7) == device.JOINT_MOUSE
    ca, cb = contacts["bodyA"][cl].astype(np.int64), contacts["bodyB"][cl].astype(np.int64)
    raw_a, raw_b = np.concatenate([ja, ca]), np.concatenate([jb, cb])
    a = np.where(np.concatenate([mouse, np.zeros(len(ca), bool)]), -1, raw_a)
    a = np.where((a >= 0) & mov[np.maximum(a, 0)], a, -1)
    b = np.where((raw_b >= 0) & mov[np.maximum(raw_b, 0)], raw_b, -1)
    b = np.where(a == b, -1, b)
    return a, b, raw_a, raw_b


def degrees(bodies, contacts, joints):
    """Incidence-list length of every body slot (s2bItemEndpoints' degree)."""
    a, b, _, _ = item_ends(bodies, contacts, joints)
    e = np.concatenate([a[a >= 0], b[b >= 0]])
    return np.bincount(e, minlength=len(bodies))


def serial_sizes(bodies, contacts, joints, hub_degree=HUB_DEGREE):
    """(contacts, joints, distinct bodies) of the serial overflow group when every constraint of a body above `hub_degree`
    (> 0) goes there uncoloured and no other constraint runs out of colours (the scenes here are stars: only a hub's
    constraints conflict, so a caller whose hub runs out of colours adds those itself)."""
    a, b, raw_a, raw_b = item_ends(bodies, contacts, joints)
    deg = degrees(bodies, contacts, joints)
    hub = np.zeros(len(a), bool)
    for e in (a, b):
        hub |= (e >= 0) & (deg[np.maximum(e, 0)] > hub_degree) & (hub_degree > 0)  # 0: every constraint is coloured
    nj = int(((joints["flags"] & 1) == 1).sum())
    ends = np.concatenate([raw_a[hub], raw_b[hub]])
    return int(hub[nj:].sum()), int(hub[:nj].sum()), len(np.unique(ends[ends >= 0]))


def hub_lists(bodies, contacts, joints):
    deg = degrees(bodies, contacts, joints)
    return sorted(deg[deg > HEAVY_DEGREE].tolist())


def check_sizes(name, bodies, contacts, joints):
    """Assert the sizes SCENES lists for `name` on its rows (CPU and GPU tests alike)."""
    _, want = SCENES[name]
    deg = degrees(bodies, contacts, joints)
    assert hub_lists(bodies, contacts, joints) == sorted(want["hubs"]), (name, hub_lists(bodies, contacts, joints))
    if "serial" in want:
        assert serial_sizes(bodies, contacts, joints) == want["serial"], (name, serial_sizes(bodies, contacts, joints))
    for n in set(want.get("lists", [])):
        assert int((deg == n).sum()) >= want["lists"].count(n), (name, n, int((deg == n).sum()))
    return deg
