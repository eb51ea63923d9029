"""GPU: neighbour-synchronised colour steps of the persistent solver kernel (DESIGN.md §3.1).

Block b runs the b-th share of every device-wide colour; between two colour steps it waits only for the blocks that run
constraints sharing a movable body with its own (its neighbours), not for the whole grid. The solve order does not change,
so a world stepped with the mode on must match, bit for bit, the same world stepped with a grid barrier before every colour
step (S2B_NEIGHBOUR_SYNC=0), for every variant. The other parity tests replay the oracle in the order the device reports and
cover the mode wherever the device turns it on."""
import os

import numpy as np
import pytest

from solver2d_b200 import capi, device, scenes

pytestmark = pytest.mark.gpu
DT = 1.0 / 60.0


@pytest.fixture(scope="module")
def product():
    return capi.Solver2D(device.LIB_PATH)


@pytest.fixture(scope="module")
def dev():
    return device.Device()


def _build(product, dev, recipe, solver, neighbour_sync, regions=None, restitution=False, **kw):
    """A scene pushed to the device with the mode allowed (the device decides) or switched off."""
    old = os.environ.get("S2B_NEIGHBOUR_SYNC")
    os.environ["S2B_NEIGHBOUR_SYNC"] = "1" if neighbour_sync else "0"
    try:
        sc = recipe(product, solver, **kw)
        dev.lib.s2World_Flush.restype = None
        dev.lib.s2World_Flush.argtypes = [capi.WorldId]
        dev.lib.s2World_Flush(sc.world)
        dw = device.DeviceWorld.attach(dev, sc.world)
    finally:
        if old is None:
            del os.environ["S2B_NEIGHBOUR_SYNC"]
        else:
            os.environ["S2B_NEIGHBOUR_SYNC"] = old
    if regions is not None:
        dw.set_regions(regions)
    if restitution:
        dw.set_restitution(True)
    return sc, dw


def _state(dw):
    c = dw.counters()
    return (dw.download_all_bodies().view(np.uint8), dw.download_contacts(c.contactCount + 64).view(np.uint8),
            dw.download_joints().view(np.uint8))


# Every scene has more than 1 024 bodies, so the persistent kernel runs on several blocks, and regions are off, so every
# colour is a device-wide step: the mode has to come on in each of them (asserted below). (recipe, arguments, options, steps,
# whether the constraint set must change during the run)
SCENES = {
    # a multistep pile
    "pyramid": (scenes.pyramid, dict(base_count=48), dict(), 24, False),
    # 1 600 boxes dropped onto two bridges: joints and contacts share the colour steps, and the constraint set changes as the
    # boxes land (after about 60 steps) and pile up
    "bridges_boxes": (scenes.joint_contact_stress, dict(bridges=2, planks=40, grid=40), dict(), 100, True),
    # prismatic / revolute / mouse joints, boxes riding kinematic carriages (kinematic endpoints make no neighbour edge)
    "kinematic": (scenes.sliders, dict(copies=56), dict(), 40, False),
    # restitution on (its own kernel continues the epochs), layers of shapes landing one after another, a kinematic platform
    "restitution": (scenes.bouncers, dict(columns=48, rows=24), dict(restitution=True), 80, True),
}


@pytest.mark.parametrize("scene", list(SCENES))
@pytest.mark.parametrize("solver", capi.SOLVER_TYPES)
def test_neighbour_sync_bit_identical_to_grid_barriers(product, dev, solver, scene):
    recipe, kw, opts, steps, churn = SCENES[scene]
    on, dw_on = _build(product, dev, recipe, solver, True, regions=0, **opts, **kw)
    off, dw_off = _build(product, dev, recipe, solver, False, regions=0, **opts, **kw)
    used = 0
    constraint_counts = set()
    try:
        for step in range(steps):
            on.step(DT, 4, 2, True)
            off.step(DT, 4, 2, True)
            c = dw_on.counters()
            assert dw_off.counters().neighbourSync == 0
            used += c.neighbourSync > 1
            constraint_counts.add(c.constraintCount)
            for what, a, b in zip(("bodies", "contacts", "joints"), _state(dw_on), _state(dw_off)):
                assert np.array_equal(a, b), f"step {step}: {what} differ with neighbour-synchronised colour steps"
    finally:
        on.destroy()
        off.destroy()
    assert used > steps // 2, f"the neighbour-synchronised colour steps ran in only {used} of {steps} steps"
    if churn:
        assert len(constraint_counts) > 2, "the constraint set never changed"


def test_mode_decided_on_device(product, dev):
    """On for the 100 128- and 5 050-box pyramids, off for the tumbler (a hub: its constraints go to the serial group)."""
    for base in (447, 100):
        sc, dw = _build(product, dev, scenes.pyramid, "TGS_Soft", True, base_count=base)
        try:
            for _ in range(3):
                sc.step(DT, 4, 2, True)
            c = dw.counters()
            assert c.regionCount == 0 and c.neighbourSync > 1, f"pyramid {base}: mode off ({c.neighbourSync})"
        finally:
            sc.destroy()
    sc, dw = _build(product, dev, scenes.tumbler, "TGS_Soft", True, grid=60)
    try:
        # (the boxes first fall onto the container's floor; the hub's constraints appear once they touch it)
        for _ in range(200):
            sc.step(DT, 4, 2, True)
            c = dw.counters()
            if c.overflowCount > 0:
                break
        assert c.overflowCount > 0 and c.neighbourSync == 0
    finally:
        sc.destroy()


@pytest.mark.parametrize("base", [40, 100])
def test_constraints_sharing_a_body_run_on_neighbours(product, dev, base):
    """On the downloaded tables: every two constraints that share a movable body run on the same block or on neighbours."""
    sc, dw = _build(product, dev, scenes.pyramid, "TGS_Soft", True, regions=0, base_count=base)
    try:
        for _ in range(6):
            sc.step(DT, 4, 2, True)
        nbrs = dw.neighbour_blocks()
        blocks = len(nbrs)
        assert blocks > 1
        for b, row in enumerate(nbrs):
            assert len(row) <= 16 and b not in row and all(b in nbrs[o] for o in row), f"block {b}: list not symmetric"
        c = dw.counters()
        order, sizes = dw.solve_order(c.constraintCount + c.jointCount + 16, max_groups=200)
        assert sizes.sum() == len(order) == c.constraintCount + c.jointCount
        contacts = dw.download_contacts(c.contactCount + 64)
        joints = dw.download_joints()
        bodies = dw.download_all_bodies()
        movable = (bodies["invMass"] != 0) | (bodies["invI"] != 0)
        touched = {}
        pos = 0
        for n in sizes.tolist():
            share = ((n + blocks - 1) // blocks + 31) // 32 * 32
            for u in range(n):
                item = int(order[pos + u])
                row = contacts[item] if item >= 0 else joints[-1 - item]
                for body in (int(row["bodyA"]), int(row["bodyB"])):
                    if body >= 0 and movable[body]:
                        touched.setdefault(body, set()).add(u // share)
            pos += n
        for body, owners in touched.items():
            for x in owners:
                for y in owners:
                    assert x == y or y in nbrs[x], f"body {body}: blocks {x} and {y} are not neighbours"
    finally:
        sc.destroy()
