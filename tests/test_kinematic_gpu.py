"""GPU: kinematic bodies under all ten variants and every schedule, every step against the reference pipeline.

scenes.kinematic_rigs: piles on sliding kinematic platforms and a turntable, pendulums, sliders and motorised cranks on
moving, turning kinematic carriages, a mouse joint — several thread blocks of constraints. The harness is the one of
test_multistep_gpu (reference collide, the prismatic oracle in the device's order, reference finalize) with the delta
position carried from step to step: XPBD never resets a kinematic body's (DESIGN.md §3.8), and the device's is compared
with the oracle's every step next to the bodies, manifolds and joint impulses. Welds on a kinematic platform are checked
the same way in test_weld_gpu.

Mutations each test catches: a delta position dropped when the host re-uploads a kinematic body's row (a velocity setter
between steps) fails test_public_api_drive_* under XPBD; a kinematic body's delta position reset by XPBD's finalize, or
left out of the contact and joint rows, fails test_every_step under XPBD in every mode."""
import ctypes as C

import numpy as np
import pytest

import joint_oracle
from helpers import bit_equal
from oracle import ref as refmod
from solver2d_b200 import capi, device, scenes
from test_e2e_gpu import _angles, _positions, _ref_pair_table
from test_first_touch_warm_gpu import GATHER_CODE, SUBSTEPS, _trace
from test_multistep_gpu import _run, _steps
from test_prismatic_gpu import _as_prismatic, _slots

pytestmark = pytest.mark.gpu
DT = 1.0 / 60.0
VARIANTS = ["Jacobi", "PGS", "PGS_NGS", "PGS_NGS_Block", "PGS_Soft", "SoftStep", "TGS_Sticky", "TGS_Soft", "TGS_NGS", "XPBD"]
KW = dict(platforms=4, base_count=12)


@pytest.fixture(scope="module")
def product():
    return capi.Solver2D(device.LIB_PATH)


def _as_joints(joints, sc):
    return _as_prismatic(joints, _slots(sc), sc.piles["prismatic_defs"])


class _Seen:
    """The largest value of each schedule counter over the checked steps."""

    def __init__(self):
        self.max = {}

    def __call__(self, dw):
        c = dw.counters()
        for name in ("constraintCount", "regionCount", "cutCount", "neighbourSync", "overflowCount"):
            self.max[name] = max(self.max.get(name, 0), getattr(c, name))


# mode: (device setup, what the counters must show)
MODES = {
    "default": (None, lambda m: True),
    "regions": (lambda dw: dw.set_regions(2), lambda m: m["regionCount"] >= 2 and m["cutCount"] > 0),
    "no_regions": (lambda dw: dw.set_regions(0), lambda m: m["regionCount"] == 0 and m["neighbourSync"] > 1),
    "overflow": (lambda dw: dw.set_max_colors(2), lambda m: m["overflowCount"] > 0),
}


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("solver", VARIANTS)
def test_every_step(reference, product, dev, solver, mode):
    setup, ran = MODES[mode]
    seen = _Seen()
    _run(reference, product, dev, scenes.kinematic_rigs, solver, _steps(solver, 30), 4, 2, KW, setup=setup,
         oracle=joint_oracle.load(), as_joints=_as_joints, after_step=seen)
    assert seen.max["constraintCount"] > 512, seen.max
    assert ran(seen.max), f"{mode}: the schedule did not run as asked: {seen.max}"


def _drive(turn):
    """Public-API calls on both worlds: every five steps new velocities for every kinematic body; once, a shape added to a
    platform."""
    def before_step(step, worlds):
        for lib, sc in worlds:
            if step % 5 == 2:
                for k, bid in enumerate(sc.piles["kinematic"]):
                    sign = 1.0 if (k + step // 5) % 2 == 0 else -1.0
                    lib.s2Body_SetLinearVelocity(bid, capi.Vec2(sign * (0.3 + 0.05 * k), 0.02 * (step % 3)))
                    lib.s2Body_SetAngularVelocity(bid, sign * 0.2 if turn else 0.0)
            if step == 13:
                sd = capi.default_shape_def()
                sd.density = 1.0
                box = lib.s2MakeOffsetBox(0.5, 0.5, capi.Vec2(5.0, 1.0), 0.0)
                lib.s2CreatePolygonShape(sc.piles["kinematic"][0], C.byref(sd), C.byref(box))
    return before_step


@pytest.mark.parametrize("solver", VARIANTS)
def test_public_api_drive_every_step(reference, product, dev, solver):
    """Velocity setters on the kinematic bodies every few steps and a shape added to one: each re-uploads the body's row.
    Every step against the reference pipeline replayed in the device's order."""
    _run(reference, product, dev, scenes.kinematic_rigs, solver, _steps(solver, 30), 4, 2, KW, oracle=joint_oracle.load(),
         as_joints=_as_joints, before_step=_drive(True))


@pytest.mark.parametrize("solver", VARIANTS)
def test_public_api_drive_reference_order(reference, product, dev, solver):
    """The same drive, the reference library running free and the device in the reference's order (wavefront schedule,
    the reference's contact order): positions and angles bit for bit after every step. Revolute stand-ins on both sides
    (the reference has no prismatic joint); the kinematic bodies do not turn, because the reference's position passes
    renormalise a turning kinematic body's rotation at every constraint on it (DESIGN.md §3.8)."""
    R, P = reference, product
    kw = dict(KW, prismatic=False, turning=False)
    sr = scenes.kinematic_rigs(R, solver, **kw)
    sp = scenes.kinematic_rigs(P, solver, **kw)
    dw = device.DeviceWorld.attach(dev, sp.world)
    dw.set_schedule(device.SCHEDULE_WAVEFRONT)
    drive = _drive(False)
    try:
        for step in range(_steps(solver, 30)):
            drive(step, ((R, sr), (P, sp)))
            R.step_collide(sr.world)
            keys, *_ = _ref_pair_table(R, sr.world)
            dw.set_contact_order(keys)
            R.step_solve(sr.world, DT, 4, 2, True)
            R.step_finalize(sr.world)
            sp.step(DT, 4, 2, True)
            assert np.array_equal(_positions(R, sr), _positions(P, sp)), f"{solver} step {step}: positions"
            assert np.array_equal(_angles(R, sr), _angles(P, sp)), f"{solver} step {step}: angles"
        bf, bi = R.bodies(sr.world)
        F = refmod.BODY_F
        v = bi[:, 0] == 1
        assert bit_equal(dw.download_delta_positions(len(bf))[v], bf[v, F["dp"]:F["dp"] + 2])
        assert dw.counters().constraintCount > (0 if solver == "Jacobi" else 512)  # Jacobi's piles are apart after 12 steps
    finally:
        sr.destroy()
        sp.destroy()


def test_tgs_soft_gather_pass_kept_every_step(reference, product, dev):
    """TGS_Soft with the warm start at the first touch: a contact on a kinematic body keeps the per-sub-step gather pass.
    That path, regions off, every step against the reference pipeline."""
    sc = scenes.kinematic_rigs(product, "TGS_Soft", **KW)
    try:
        dw = device.DeviceWorld.attach(dev, sc.world)
        dw.set_regions(0)
        for _ in range(3):
            sc.step(DT, SUBSTEPS, 2, True)
        assert _trace(dev, dw, sc).count(GATHER_CODE) == SUBSTEPS
    finally:
        sc.destroy()
    seen = _Seen()
    _run(reference, product, dev, scenes.kinematic_rigs, "TGS_Soft", 40, SUBSTEPS, 2, KW, setup=lambda dw: dw.set_regions(0),
         oracle=joint_oracle.load(), as_joints=_as_joints, after_step=seen)
    assert seen.max["regionCount"] == 0 and seen.max["neighbourSync"] > 1, seen.max
