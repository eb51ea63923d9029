"""GPU: contact rows of the solver's constraint stream written by the narrow phase (DESIGN.md §3.4).

While the solve schedule stands, each narrow-phase thread writes its constraint's row itself (s2bWriteContactRow) and the
persistent solver kernel skips the contact part of its prepare pass. A step that rebuilds the schedule prepares every row in
the kernel as before. Same values, same arithmetic: every scene must match, bit for bit and after every step, the same scene
stepped with S2B_NARROWPHASE_PREPARE=0 (prepare gathers every row). The counter narrowphaseRowSteps must advance on the steps
that use the rows and stay put on the steps that rebuild the schedule."""
import ctypes as C
import os

import numpy as np
import pytest

from solver2d_b200 import capi, device, scenes
from solver2d_b200.capi import Vec2, default_body_def, default_shape_def

pytestmark = pytest.mark.gpu
DT = 1.0 / 60.0

# variants whose program prepares contacts with s2bPrepareContact (COP_PREPARE / COP_PREPARE_COLD)
COVERED = ["Jacobi", "PGS", "PGS_NGS", "PGS_Soft", "SoftStep", "TGS_Soft", "TGS_NGS", "XPBD"]
# variants with a prepare of their own: the narrow phase never writes their rows
NOT_COVERED = ["TGS_Sticky", "PGS_NGS_Block"]


@pytest.fixture(scope="module")
def product():
    return capi.Solver2D(device.LIB_PATH)


@pytest.fixture(scope="module")
def dev():
    return device.Device()


def _build(product, dev, recipe, solver, enabled, regions=None):
    old = os.environ.get("S2B_NARROWPHASE_PREPARE")
    os.environ["S2B_NARROWPHASE_PREPARE"] = "1" if enabled else "0"
    try:
        sc = recipe(product, solver)
        dev.lib.s2World_Flush.restype = None
        dev.lib.s2World_Flush.argtypes = [capi.WorldId]
        dev.lib.s2World_Flush(sc.world)
        dw = device.DeviceWorld.attach(dev, sc.world)
    finally:
        if old is None:
            del os.environ["S2B_NARROWPHASE_PREPARE"]
        else:
            os.environ["S2B_NARROWPHASE_PREPARE"] = old
    if regions is not None:
        dw.set_regions(regions)
    return sc, dw


def _state(dw):
    c = dw.counters()
    return dw.download_all_bodies().view(np.uint8), dw.download_contacts(c.contactCount + 64).view(np.uint8)


def _pyramid(base):
    return lambda lib, solver: scenes.pyramid(lib, solver, base_count=base)


def _resting_stacks(lib, solver):
    """Stacks of one, two and three boxes resting on the ground, apart from each other: steady under every variant (a
    Jacobi pyramid slides apart, and its set of live constraints changes every step)."""
    sc = scenes.pyramid(lib, solver, base_count=1)
    bd = default_body_def()
    bd.type = capi.DYNAMIC_BODY
    sd = default_shape_def()
    sd.density = 1.0
    box = lib.s2MakeSquare(0.5)
    for k in range(48):
        for level in range(1 + k % 3):
            bd.position = Vec2(-61.25 + 2.5 * k, 0.5 + 1.0 * level)
            bid = lib.s2CreateBody(sc.world, C.byref(bd))
            lib.s2CreatePolygonShape(bid, C.byref(sd), C.byref(box))
            sc.bodies.append(bid)
    return sc


def _pile_with_droppers(lib, solver):
    """A pyramid with rows of boxes above it that fall in one after another: contacts gain and lose points, and the pair pass
    merges new pairs into the contact table."""
    sc = scenes.pyramid(lib, solver, base_count=16)
    bd = default_body_def()
    bd.type = capi.DYNAMIC_BODY
    sd = default_shape_def()
    sd.density = 1.0
    box = lib.s2MakeSquare(0.5)
    for row in range(4):
        for k in range(10):
            bd.position = Vec2(-7.25 + 1.5 * k + 0.25 * row, 18.0 + 3.0 * row)
            bd.angularVelocity = 0.2 * ((k % 3) - 1)
            bid = lib.s2CreateBody(sc.world, C.byref(bd))
            lib.s2CreatePolygonShape(bid, C.byref(sd), C.byref(box))
            sc.bodies.append(bid)
    return sc


def _pile_with_platform(lib, solver):
    """A pyramid and, away from it, a kinematic platform sliding sideways with a stack of boxes resting on it."""
    sc = scenes.pyramid(lib, solver, base_count=20)
    kd = default_body_def()
    kd.type = capi.KINEMATIC_BODY
    kd.position = Vec2(40.0, 4.0)
    kd.linearVelocity = Vec2(0.8, 0.0)
    pid = lib.s2CreateBody(sc.world, C.byref(kd))
    sd = default_shape_def()
    sd.density = 1.0
    lib.s2CreatePolygonShape(pid, C.byref(sd), C.byref(lib.s2MakeBox(6.0, 0.25)))
    sc.bodies.append(pid)
    bd = default_body_def()
    bd.type = capi.DYNAMIC_BODY
    box = lib.s2MakeSquare(0.5)
    for i in range(5):
        for j in range(6):
            bd.position = Vec2(37.5 + 1.0 * j, 4.75 + 1.0 * i)
            bid = lib.s2CreateBody(sc.world, C.byref(bd))
            lib.s2CreatePolygonShape(bid, C.byref(sd), C.byref(box))
            sc.bodies.append(bid)
    return sc


def _field(lib, solver):
    return scenes.pyramid_field(lib, solver, count=24, base_count=6)


def _run(on, dw_on, off, dw_off, steps, warm=lambda step: True, between=None):
    """Steps both worlds, compares them after every step; returns, per step, (rows counter advance, live constraints)."""
    history = []
    before = dw_on.counters().narrowphaseRowSteps
    for step in range(steps):
        if between is not None:
            between(step, dw_on)
            between(step, dw_off)
        on.step(DT, 4, 2, warm(step))
        off.step(DT, 4, 2, warm(step))
        for what, a, b in zip(("bodies", "contacts"), _state(dw_on), _state(dw_off)):
            assert np.array_equal(a, b), f"step {step}: {what} differ with the contact rows written by the narrow phase"
        c = dw_on.counters()
        history.append((c.narrowphaseRowSteps - before, c.constraintCount))
        before = c.narrowphaseRowSteps
        assert dw_off.counters().narrowphaseRowSteps == 0
    return history


def _check_counter(history, min_used):
    used = sum(d for d, _ in history)
    assert all(d in (0, 1) for d, _ in history), history
    # a step whose live-constraint count changed has rebuilt the schedule: its rows came from prepare
    for k in range(1, len(history)):
        if history[k][1] != history[k - 1][1]:
            assert history[k][0] == 0, (k, history)
    assert used >= min_used, (used, history)


def _pair(product, dev, recipe, solver, **opts):
    on, dw_on = _build(product, dev, recipe, solver, True, **opts)
    off, dw_off = _build(product, dev, recipe, solver, False, **opts)
    return on, dw_on, off, dw_off


@pytest.mark.parametrize("solver", COVERED)
def test_steady_scene_bit_identical(product, dev, solver):
    on, dw_on, off, dw_off = _pair(product, dev, _resting_stacks, solver)
    try:
        history = _run(on, dw_on, off, dw_off, 16)
        # steps 1 and 2 are eager (no graph yet); from then on a standing schedule takes the narrow phase's rows
        _check_counter(history, 8)
    finally:
        on.destroy()
        off.destroy()


@pytest.mark.parametrize("solver", COVERED)
def test_pyramid_bit_identical(product, dev, solver):
    """A pyramid under every covered variant: steady under most, sliding apart under some (the counter then only has to
    stay put on the rebuild steps)."""
    on, dw_on, off, dw_off = _pair(product, dev, _pyramid(30), solver)
    try:
        history = _run(on, dw_on, off, dw_off, 16)
        _check_counter(history, 0)
    finally:
        on.destroy()
        off.destroy()


@pytest.mark.parametrize("solver", NOT_COVERED)
def test_variants_with_their_own_prepare_never_take_rows(product, dev, solver):
    on, dw_on, off, dw_off = _pair(product, dev, _pyramid(20), solver)
    try:
        history = _run(on, dw_on, off, dw_off, 8)
        assert sum(d for d, _ in history) == 0
    finally:
        on.destroy()
        off.destroy()


def test_boxes_dropping_into_a_pile(product, dev):
    on, dw_on, off, dw_off = _pair(product, dev, _pile_with_droppers, "TGS_Soft")
    try:
        history = _run(on, dw_on, off, dw_off, 90)
        _check_counter(history, 10)
        # the droppers landed: the live set changed along the way
        assert len({n for _, n in history}) > 3
    finally:
        on.destroy()
        off.destroy()


def test_a_step_without_warm_start(product, dev):
    for solver in ("TGS_Soft", "PGS"):
        on, dw_on, off, dw_off = _pair(product, dev, _resting_stacks, solver)
        try:
            history = _run(on, dw_on, off, dw_off, 14, warm=lambda step: step != 8)
            _check_counter(history, 5)
            # other step settings: rebuilt eagerly, and once more when the graph's settings come back
            assert history[8][0] == 0 and history[9][0] == 0
        finally:
            on.destroy()
            off.destroy()


def test_mass_change_between_steps(product, dev):
    """A box's mass and inertia change on the device between two steps (it stays dynamic, so the schedule may stand)."""

    def heavier(step, dw):
        if step != 6:
            return
        rows = dw.download_all_bodies()
        k = int(np.flatnonzero(rows["invMass"] > 0)[len(rows) // 3])
        row = rows[k:k + 1].copy()
        row["mass"] *= 3.0
        row["I"] *= 3.0
        row["invMass"] = 1.0 / row["mass"]
        row["invI"] = 1.0 / row["I"]
        dw.upload_bodies(row, dw.body_cap)

    on, dw_on, off, dw_off = _pair(product, dev, _resting_stacks, "TGS_Soft")
    try:
        history = _run(on, dw_on, off, dw_off, 14, between=heavier)
        _check_counter(history, 5)
    finally:
        on.destroy()
        off.destroy()


def test_kinematic_platform_carrying_boxes(product, dev):
    on, dw_on, off, dw_off = _pair(product, dev, _pile_with_platform, "TGS_Soft", regions=0)
    try:
        history = _run(on, dw_on, off, dw_off, 30)
        _check_counter(history, 10)
    finally:
        on.destroy()
        off.destroy()


def test_resident_region_field(product, dev):
    on, dw_on, off, dw_off = _pair(product, dev, _field, "TGS_Soft")
    try:
        history = _run(on, dw_on, off, dw_off, 24)
        assert dw_on.counters().regionCount > 0 and dw_off.counters().regionCount > 0
        _check_counter(history, 8)
    finally:
        on.destroy()
        off.destroy()
