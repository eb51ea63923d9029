"""CPU: kinematic bodies in the oracle, pinned against the UNMODIFIED reference every step, for all ten variants.

XPBD finalises dynamic bodies only (reference src/solve_xpbd.c:497-511): a kinematic body's deltaPosition is never added to
its position nor reset, so it grows from step to step while its position stays where it was created, and every contact and
joint row on the body reads it (src/solve_xpbd.c:113, src/revolute_joint.c:268,314). The oracle takes the deltaPosition
each body starts the stage with and returns the one the stage leaves (port.Oracle.solve(..., dp=...)); the every-step GPU
harnesses carry it from step to step that way. Here the reference runs free, and at every step the oracle is run from the
reference's state, deltaPosition included, against the reference's own solver stage."""
import numpy as np
import pytest

from helpers import bit_equal, body_rows_from_ref, contact_rows_from_ref, joint_rows_from_ref, ref_delta_positions
from oracle import port
from oracle import ref as refmod
from solver2d_b200 import capi, device, scenes

DT = 1.0 / 60.0
VARIANTS = ["Jacobi", "PGS", "PGS_NGS", "PGS_NGS_Block", "PGS_Soft", "SoftStep", "TGS_Sticky", "TGS_Soft", "TGS_NGS", "XPBD"]


def _pin_every_step(R, solver, steps, carry_dp=True, turning=False):
    """Runs `steps` reference steps; before each solver stage, the oracle from the reference's state. Returns the largest
    |deltaPosition| the kinematic bodies started a stage with."""
    O = port.load()
    sc = scenes.kinematic_rigs(R, solver, platforms=2, base_count=6, turning=turning)
    ctx = device.make_context(solver, DT, 4, 2, True)
    F = refmod.BODY_F
    kinematic = np.array([b.index for b in sc.piles["kinematic"]])
    carried = 0.0
    try:
        for step in range(steps):
            R.step_collide(sc.world)
            bf, bi = R.bodies(sc.world)
            contacts, slots = contact_rows_from_ref(*R.contacts(sc.world))
            joints = joint_rows_from_ref(*R.joints(sc.world))
            dp = ref_delta_positions(R, sc.world) if carry_dp else np.zeros((len(bf), 2), dtype=np.float32)
            carried = max(carried, float(np.abs(ref_delta_positions(R, sc.world)[kinematic]).max()))
            ob, oc, oj, odp = O.solve(capi.SOLVER[solver], body_rows_from_ref(bf, bi), contacts, joints, ctx, dp=dp)

            R.step_solve(sc.world, DT, 4, 2, True)
            bf2, bi2 = R.bodies(sc.world)
            valid = bi2[:, 0] == 1
            for name, col, width in (("position", F["position"], 2), ("rot", F["rot"], 2), ("linearVelocity", F["v"], 2)):
                assert bit_equal(ob[name][valid], bf2[valid, col:col + width]), f"{solver} step {step}: {name}"
            assert bit_equal(ob["angularVelocity"][valid], bf2[valid, F["w"]]), f"{solver} step {step}: angularVelocity"
            assert bit_equal(odp[valid], bf2[valid, F["dp"]:F["dp"] + 2]), f"{solver} step {step}: deltaPosition"
            cf2, _ = R.contacts(sc.world)
            P = refmod.POINT_F
            for j in range(2):
                base = refmod.CONTACT_F["points"] + refmod.POINT_STRIDE * j
                live = oc["pointCount"] > j
                for name in ("normalImpulse", "tangentImpulse"):
                    assert bit_equal(oc["points"][name][:, j][live], cf2[slots, base + P[name]][live]), \
                        f"{solver} step {step}: {name}"
            want = joint_rows_from_ref(*R.joints(sc.world))
            jv = (want["flags"] & 1) == 1
            for name in ("impulse", "motorImpulse", "lowerImpulse", "upperImpulse"):
                assert bit_equal(oj[name][jv], want[name][jv]), f"{solver} step {step}: joint {name}"
            R.step_finalize(sc.world)
    finally:
        sc.destroy()
    return carried


@pytest.mark.parametrize("solver", VARIANTS)
def test_kinematic_rigs_every_step_pinned(reference, solver):
    """Piles on sliding platforms, revolute and stand-in prismatic joints from moving carriages, a mouse joint: 40 steps
    (Jacobi, which blows piles apart in the reference too, 12)."""
    carried = _pin_every_step(reference, solver, 12 if solver == "Jacobi" else 40)
    if solver == "XPBD":
        # the kinematic bodies' deltaPosition really was carried: 40 steps at 0.4 to 0.6 m/s
        assert carried > 0.2, carried
    else:
        assert carried == 0.0, carried


def test_xpbd_needs_the_carried_delta_position(reference):
    """Without the deltaPosition carried in, XPBD's stage differs from the reference's from the second step on."""
    with pytest.raises(AssertionError, match="step 1:"):
        _pin_every_step(reference, "XPBD", 3, carry_dp=False)


@pytest.mark.parametrize("solver", ["Jacobi", "PGS", "PGS_Soft", "SoftStep", "TGS_Sticky", "TGS_Soft"])
def test_turning_kinematic_bodies_every_step_pinned(reference, solver):
    """The carriages and a turntable also turn. Only the variants without a position-level pass: the reference's position
    passes write a kinematic body's rotation back renormalised at every constraint on it (DESIGN.md §3.8)."""
    _pin_every_step(reference, solver, 12 if solver == "Jacobi" else 40, turning=True)
