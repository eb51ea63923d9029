"""GPU: the TGS_Soft warm start run at each body's first constraint of the bias sweep (DESIGN.md §3.1).

Where the bias sweep integrates positions at a body's last constraint, it also runs the warm-start gather of a body just before
the body's first constraint, and the per-sub-step gather pass with its grid barriers goes away. Bodies without a constraint are
sub-stepped by the finalize pass instead. A constraint that reads a kinematic body keeps the gather pass. The operations and
their order are unchanged, so every scene must match, bit for bit and after every step, the same scene stepped with the
position folding and the gather at first touch switched off (S2B_FUSE_POSITIONS=0: both body passes)."""
import ctypes as C
import os

import numpy as np
import pytest

from solver2d_b200 import capi, device, scenes
from solver2d_b200.capi import Vec2, default_body_def, default_shape_def

pytestmark = pytest.mark.gpu
DT = 1.0 / 60.0
SUBSTEPS = 4
# trace code of the warm-start body pass: PASS_BODY << 8 | BOP_INTEGRATE_VELOCITIES_WARM (program.cuh)
GATHER_CODE = 9
START_CODE = 0xFFFF


@pytest.fixture(scope="module")
def product():
    return capi.Solver2D(device.LIB_PATH)


@pytest.fixture(scope="module")
def dev():
    return device.Device()


def _free_boxes(lib, sc, count=64):
    """Boxes high above everything, spinning and drifting apart: no constraint touches them during the run."""
    bd = default_body_def()
    bd.type = capi.DYNAMIC_BODY
    sd = default_shape_def()
    sd.density = 1.0
    box = lib.s2MakeSquare(0.25)
    for k in range(count):
        bd.position = Vec2(-80.0 + 2.5 * k, 400.0 + 3.0 * (k % 5))
        bd.linearVelocity = Vec2(0.5 * ((k % 7) - 3), 1.0 + 0.25 * (k % 3))
        bd.angularVelocity = 0.3 * ((k % 5) - 2)
        bid = lib.s2CreateBody(sc.world, C.byref(bd))
        lib.s2CreatePolygonShape(bid, C.byref(sd), C.byref(box))
        sc.bodies.append(bid)
    # a kinematic body that touches nothing either: moved by finalize too
    kd = default_body_def()
    kd.type = capi.KINEMATIC_BODY
    kd.position = Vec2(150.0, 300.0)
    kd.linearVelocity = Vec2(0.0, 0.75)
    kd.angularVelocity = 0.5
    kid = lib.s2CreateBody(sc.world, C.byref(kd))
    lib.s2CreatePolygonShape(kid, C.byref(sd), C.byref(lib.s2MakeBox(1.0, 0.2)))
    sc.bodies.append(kid)


def _platform_pile(lib, sc, columns=6, rows=6):
    """A kinematic platform sliding sideways, away from the pyramid, with a stack of boxes resting on it."""
    kd = default_body_def()
    kd.type = capi.KINEMATIC_BODY
    kd.position = Vec2(70.0, 4.0)
    kd.linearVelocity = Vec2(0.8, 0.0)
    pid = lib.s2CreateBody(sc.world, C.byref(kd))
    sd = default_shape_def()
    sd.density = 1.0
    lib.s2CreatePolygonShape(pid, C.byref(sd), C.byref(lib.s2MakeBox(6.0, 0.25)))
    sc.bodies.append(pid)
    bd = default_body_def()
    bd.type = capi.DYNAMIC_BODY
    box = lib.s2MakeSquare(0.5)
    for i in range(rows):
        for j in range(columns):
            bd.position = Vec2(70.0 - 0.5 * columns + 1.0 * j + 0.5, 4.25 + 0.5 + 1.0 * i)
            bid = lib.s2CreateBody(sc.world, C.byref(bd))
            lib.s2CreatePolygonShape(bid, C.byref(sd), C.byref(box))
            sc.bodies.append(bid)


def _pile_with_free_boxes(lib, solver):
    sc = scenes.pyramid(lib, solver, base_count=48)
    _free_boxes(lib, sc)
    return sc


def _pile_with_platform(lib, solver):
    sc = scenes.pyramid(lib, solver, base_count=48)
    _platform_pile(lib, sc)
    return sc


def _build(product, dev, recipe, fuse, restitution=False, regions=None):
    old = os.environ.get("S2B_FUSE_POSITIONS")
    os.environ["S2B_FUSE_POSITIONS"] = "1" if fuse else "0"
    try:
        sc = recipe(product, "TGS_Soft")
        dev.lib.s2World_Flush.restype = None
        dev.lib.s2World_Flush.argtypes = [capi.WorldId]
        dev.lib.s2World_Flush(sc.world)
        dw = device.DeviceWorld.attach(dev, sc.world)
    finally:
        if old is None:
            del os.environ["S2B_FUSE_POSITIONS"]
        else:
            os.environ["S2B_FUSE_POSITIONS"] = old
    if regions is not None:
        dw.set_regions(regions)
    if restitution:
        dw.set_restitution(True)
    return sc, dw


def _state(dw):
    c = dw.counters()
    return dw.download_all_bodies().view(np.uint8), dw.download_contacts(c.contactCount + 64).view(np.uint8)


def _trace(dev, dw, sc):
    """The persistent kernel's time stamps of one step: codes, in order."""
    L = dev.lib
    L.s2b_set_solve_trace.argtypes = [C.c_void_p, C.c_int]
    L.s2b_get_solve_trace.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    L.s2b_get_solve_trace.restype = C.c_int
    L.s2b_set_solve_trace(dw.h, 1024)
    try:
        sc.step(DT, SUBSTEPS, 2, True)
        out = np.zeros(1024, dtype=np.uint64)
        n = L.s2b_get_solve_trace(dw.h, out.ctypes.data, 1024)
    finally:
        L.s2b_set_solve_trace(dw.h, 0)
    return [int(c) for c in (out[:n] >> np.uint64(48))]


def _pyramid(base, restitution=0.0):
    return lambda lib, solver: scenes.pyramid(lib, solver, base_count=base, restitution=restitution)


SCENES = {
    # the bench pile and a middle-sized one, default schedule
    "pyramid447": (_pyramid(447), dict(), 30),
    "pyramid100": (_pyramid(100), dict(), 30),
    # bodies without any constraint: sub-stepped by the finalize pass
    "free_boxes": (_pile_with_free_boxes, dict(regions=0), 30),
    # a constraint reads a kinematic body: the warm-start pass stays
    "platform": (_pile_with_platform, dict(regions=0), 40),
    # restitution on (its pass runs after the variant's kernel)
    "pyramid447_restitution": (_pyramid(447, restitution=0.3), dict(restitution=True), 30),
}


@pytest.mark.parametrize("scene", list(SCENES))
def test_first_touch_warm_start_bit_identical_to_body_passes(product, dev, scene):
    recipe, opts, steps = SCENES[scene]
    on, dw_on = _build(product, dev, recipe, True, **opts)
    off, dw_off = _build(product, dev, recipe, False, **opts)
    try:
        for step in range(steps):
            on.step(DT, SUBSTEPS, 2, True)
            off.step(DT, SUBSTEPS, 2, True)
            for what, a, b in zip(("bodies", "contacts"), _state(dw_on), _state(dw_off)):
                assert np.array_equal(a, b), f"step {step}: {what} differ with the warm start at the first touch"
        assert dw_on.counters().regionCount == 0
    finally:
        on.destroy()
        off.destroy()


def test_no_gather_pass_and_two_grid_barriers_on_the_bench_pile(product, dev):
    """447 pyramid: no warm-start pass in the trace; every colour step after the first one of the launch is reached through a
    neighbour wait, so the launch has two grid barriers: after prepare and before finalize."""
    sc, dw = _build(product, dev, _pyramid(447), True)
    try:
        for _ in range(3):
            sc.step(DT, SUBSTEPS, 2, True)
        codes = _trace(dev, dw, sc)
        c = dw.counters()
        assert c.regionCount == 0 and c.neighbourSync > 1
        colours = c.groupCount
        assert codes.count(START_CODE) == 1, codes
        assert GATHER_CODE not in codes, codes
        # start, one stamp per grid barrier (2) or neighbour wait (every colour step but the first), end
        steps = SUBSTEPS * 2 * colours
        assert len(codes) == 1 + 2 + (steps - 1) + 1, (len(codes), colours, codes)
    finally:
        sc.destroy()


def test_kinematic_contact_keeps_the_gather_pass(product, dev):
    sc, dw = _build(product, dev, _pile_with_platform, True, regions=0)
    try:
        for _ in range(3):
            sc.step(DT, SUBSTEPS, 2, True)
        codes = _trace(dev, dw, sc)
        assert codes.count(GATHER_CODE) == SUBSTEPS, codes
    finally:
        sc.destroy()
    sc, dw = _build(product, dev, _pile_with_free_boxes, True, regions=0)
    try:
        for _ in range(3):
            sc.step(DT, SUBSTEPS, 2, True)
        codes = _trace(dev, dw, sc)
        assert GATHER_CODE not in codes, codes
    finally:
        sc.destroy()
