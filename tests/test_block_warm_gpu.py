"""GPU: the block-wide warm start of the TGS_Soft bias sweep's colour-0 step (DESIGN.md §3.1 (d)).

Each block gathers the bodies its share of colour 0 first-touches together, from a table built with the schedule, instead of
one thread per marked row gathering its two bodies one after the other. A block whose copy of its table exceeds the
shared-memory budget keeps the per-thread gather, so both paths may mix in one launch. The float operations and their order
per body are unchanged, so every scene must match, bit for bit and after every step, the same scene stepped with the
per-thread gather (S2B_BLOCK_WARM=0), and the permuted oracle. The counter firstTable says how many blocks took the table."""
import ctypes as C
import os

import numpy as np
import pytest

from helpers import body_rows_from_ref, contact_rows_from_ref, joint_rows_from_ref
from oracle import port
from solver2d_b200 import capi, device, scenes
from solver2d_b200.capi import Vec2, default_body_def, default_shape_def

pytestmark = pytest.mark.gpu
DT = 1.0 / 60.0
SUBSTEPS = 4
# shared memory of one table slot / entry (solver_state.cuh, S2B_FT_SLOT_BYTES / S2B_FT_ENTRY_BYTES)
SLOT_BYTES, ENTRY_BYTES = 48, 20


@pytest.fixture(scope="module")
def product():
    return capi.Solver2D(device.LIB_PATH)


class _env:
    """S2B_BLOCK_WARM / S2B_BLOCK_WARM_BYTES while a world is created (the device world reads them once)."""

    def __init__(self, on, budget=None):
        self.values = {"S2B_BLOCK_WARM": "1" if on else "0", "S2B_BLOCK_WARM_BYTES": None if budget is None else str(budget)}

    def __enter__(self):
        self.old = {k: os.environ.get(k) for k in self.values}
        for k, v in self.values.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v

    def __exit__(self, *exc):
        for k, v in self.old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _build(product, dev, recipe, solver, on, budget=None, regions=0, **kw):
    with _env(on, budget):
        sc = recipe(product, solver, **kw)
        dev.lib.s2World_Flush.restype = None
        dev.lib.s2World_Flush.argtypes = [capi.WorldId]
        dev.lib.s2World_Flush(sc.world)
        dw = device.DeviceWorld.attach(dev, sc.world)
    dw.set_regions(regions)
    return sc, dw


def _state(dw):
    c = dw.counters()
    return (dw.download_all_bodies().view(np.uint8), dw.download_contacts(c.contactCount + 64).view(np.uint8),
            dw.download_joints().view(np.uint8))


def _run_pair(product, dev, recipe, solver, steps, budget=None, **kw):
    """Steps the scene with and without the table; returns the constraint counts seen and, per step, the blocks on the table."""
    on, dw_on = _build(product, dev, recipe, solver, True, budget, **kw)
    off, dw_off = _build(product, dev, recipe, solver, False, **kw)
    counts = set()
    used = []
    try:
        for step in range(steps):
            on.step(DT, SUBSTEPS, 2, True)
            off.step(DT, SUBSTEPS, 2, True)
            c = dw_on.counters()
            counts.add(c.constraintCount)
            used.append(c.firstTable)
            assert dw_off.counters().firstTable == 0
            for what, a, b in zip(("bodies", "contacts", "joints"), _state(dw_on), _state(dw_off)):
                assert np.array_equal(a, b), f"step {step}: {what} differ with the block-wide warm start"
    finally:
        on.destroy()
        off.destroy()
    return counts, used


def _table_bytes(dw, blocks):
    """Per block, the shared memory its first-touch table takes, recomputed from the solve order the device reports."""
    c = dw.counters()
    order, sizes = dw.solve_order(c.constraintCount + c.jointCount + 16, max_groups=200)
    contacts = dw.download_contacts(c.contactCount + 64)
    bodies = dw.download_all_bodies()
    movable = (bodies["invMass"] != 0) | (bodies["invI"] != 0)
    ends = [(int(contacts[o]["bodyA"]), int(contacts[o]["bodyB"])) for o in order.tolist()]
    first, degree = {}, {}
    for pos, pair in enumerate(ends):
        for body in pair:
            if body >= 0 and movable[body]:
                first.setdefault(body, pos)
                degree[body] = degree.get(body, 0) + 1
    n = int(sizes[0])
    share = ((n + blocks - 1) // blocks + 31) // 32 * 32
    out = np.zeros(blocks, dtype=np.int64)
    for body, pos in first.items():
        if pos < n:
            out[pos // share] += SLOT_BYTES + ENTRY_BYTES * degree[body]
    return out


def _pile_on_platform(lib, solver):
    """A kinematic platform under a small pile: a constraint reads a kinematic body, so the warm start stays a body pass."""
    sc = scenes.pyramid(lib, solver, base_count=60)
    kd = default_body_def()
    kd.type = capi.KINEMATIC_BODY
    kd.position = Vec2(90.0, 4.0)
    kd.linearVelocity = Vec2(0.8, 0.0)
    pid = lib.s2CreateBody(sc.world, C.byref(kd))
    sd = default_shape_def()
    sd.density = 1.0
    lib.s2CreatePolygonShape(pid, C.byref(sd), C.byref(lib.s2MakeBox(6.0, 0.25)))
    bd = default_body_def()
    bd.type = capi.DYNAMIC_BODY
    box = lib.s2MakeSquare(0.5)
    for i in range(6):
        for j in range(6):
            bd.position = Vec2(90.0 - 3.0 + 1.0 * j + 0.5, 4.75 + 1.0 * i)
            lib.s2CreatePolygonShape(lib.s2CreateBody(sc.world, C.byref(bd)), C.byref(sd), C.byref(box))
    return sc


def test_mid_size_pyramid(product, dev):
    _, used = _run_pair(product, dev, scenes.pyramid, "TGS_Soft", 30, base_count=100)
    assert min(used) > 1


@pytest.mark.parametrize("at", ["largest", "below_largest", "median"])
def test_budget_decides_per_block(product, dev, at):
    """A budget that the largest block copy just fits (every block takes the table), one byte short of it, or the median copy:
    the blocks over budget gather per thread and the others take the table, in the same launch."""
    sc, dw = _build(product, dev, scenes.pyramid, "TGS_Soft", True, base_count=100)
    try:
        for _ in range(3):
            sc.step(DT, SUBSTEPS, 2, True)
        blocks = len(dw.neighbour_blocks())
        sizes = _table_bytes(dw, blocks)
    finally:
        sc.destroy()
    assert blocks > 2 and sizes.min() < sizes.max()
    budget = {"largest": int(sizes.max()), "below_largest": int(sizes.max()) - 1, "median": int(np.median(sizes))}[at]
    expected = int((sizes <= budget).sum())
    assert at == "largest" or 0 < expected < blocks
    _, used = _run_pair(product, dev, scenes.pyramid, "TGS_Soft", 30, budget=budget, base_count=100)
    assert used == [expected] * 30


def test_kinematic_platform(product, dev):
    _, used = _run_pair(product, dev, _pile_on_platform, "TGS_Soft", 30)
    assert max(used) == 0


def test_constraint_set_changes_and_the_table_is_rebuilt(product, dev):
    """Layers of shapes landing one after another: the constraint set (and with it the schedule and the table) changes."""
    counts, used = _run_pair(product, dev, scenes.bouncers, "TGS_Soft", 80, columns=48, rows=24, joints=False, platform=False)
    assert len(counts) > 2, "the constraint set never changed"
    assert sum(u > 0 for u in used) > 40


def test_joints_keep_the_per_thread_gather(product, dev):
    """With joints the bias sweep does not warm-start at the first touch, so the table is never used."""
    _, used = _run_pair(product, dev, scenes.joint_contact_stress, "TGS_Soft", 40, bridges=2, planks=40, grid=40)
    assert max(used) == 0


@pytest.mark.parametrize("solver", [s for s in capi.SOLVER_TYPES if s != "TGS_Soft"])
def test_other_variants_unaffected(product, dev, solver):
    _, used = _run_pair(product, dev, scenes.pyramid, solver, 8, base_count=48)
    assert max(used) == 0


@pytest.mark.parametrize("budget", [None, 4096])
def test_matches_permuted_oracle(reference, dev, budget):
    """One eager TGS_Soft solve of a settled pile against the oracle replaying the order the device reports."""
    R = reference
    O = port.load()
    sc = scenes.pyramid(R, "TGS_Soft", base_count=60)
    for _ in range(10):
        sc.step(DT, SUBSTEPS, 2, True)
    R.step_collide(sc.world)
    bodies = body_rows_from_ref(*R.bodies(sc.world))
    contacts, _ = contact_rows_from_ref(*R.contacts(sc.world))
    joints = joint_rows_from_ref(*R.joints(sc.world))
    ctx = device.make_context("TGS_Soft", DT, SUBSTEPS, 2, True)
    with _env(True, budget):
        dw = dev.create_world(capi.SOLVER["TGS_Soft"])
    try:
        dw.upload_bodies(bodies, len(bodies))
        dw.upload_joints(joints, len(joints))
        dw.upload_contacts(contacts)
        dw.set_schedule(device.SCHEDULE_COLOR)
        dw.set_regions(0)
        dw.solve(ctx)
        got = dw.download_all_bodies(len(bodies))
        order, _ = dw.solve_order(len(contacts) + len(joints))
        on_table = dw.counters().firstTable
    finally:
        dw.destroy()
    sc.destroy()
    assert budget is not None or on_table > 1
    ob, _, _ = O.solve(capi.SOLVER["TGS_Soft"], bodies, contacts, joints, ctx, order=order)
    valid = (bodies["flags"] & 1) == 1
    for name in ("position", "rot", "linearVelocity", "angularVelocity"):
        g = np.ascontiguousarray(got[name][valid]).view(np.uint32)
        o = np.ascontiguousarray(ob[name][valid]).view(np.uint32)
        assert np.array_equal(g, o), f"{name}: device != permuted oracle"


def test_worlds_stepped_side_by_side_match(product, dev):
    """Two identical worlds whose steps overlap on the device, after another world was stepped and destroyed, must match bit for
    bit. A scratch array that grew used to free its old buffer with cudaFreeAsync, which does not wait for the world's stream
    when the buffer came from cudaMalloc: the other world could take the memory over while the copy of the old contents (the
    grid barrier's and the colour steps' epoch words among them) still read it."""
    for _ in range(3):
        sc, _ = _build(product, dev, scenes.pyramid, "TGS_Soft", False, base_count=100)
        for _ in range(3):
            sc.step(DT, SUBSTEPS, 2, True)
        sc.destroy()
        a, dw_a = _build(product, dev, scenes.pyramid, "TGS_Soft", False, base_count=100)
        b, dw_b = _build(product, dev, scenes.pyramid, "TGS_Soft", False, base_count=100)
        try:
            for step in range(4):
                a.step(DT, SUBSTEPS, 2, True)
                b.step(DT, SUBSTEPS, 2, True)
                assert np.array_equal(_state(dw_a)[0], _state(dw_b)[0]), f"step {step}: two identical worlds differ"
        finally:
            a.destroy()
            b.destroy()
