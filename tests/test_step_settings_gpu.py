"""GPU: the device step at step settings other than (1/60 s, 4 sub-steps, 2 relax iterations, warm starting on), with body
damping and gravity scales, and with the settings changing between steps. SETTINGS (test_step_settings_cpu, where the
oracle is pinned to the reference at each of them) reaches every hertz clamp on both sides, programs without a relax
sweep, TGS_Soft's relax-store fold with a segment run S - 1 = 0 times, a cold start and the sub-step count of BASELINE
config 2.

* Reference order: the unmodified reference running free and the device in its order (wavefront schedule, the
  reference's contact order), positions and angles bit for bit after every step, for every variant at every setting.
* Production schedule: colour schedule, persistent kernel, graph replays, every step against the oracle replayed in the
  device's order (test_multistep_gpu._run, tolerance 0), on a pyramid, scenes.damped_mix and scenes.limited_chains for
  every variant at every setting; TGS_Soft's first-touch table (damped bodies) and resident regions. The counters show the
  graph replays, the contact rows the narrow phase writes, the first-touch table and the resident regions at work.
* Settings that change mid-run: every variant, every step checked; a run of three or more equal steps replays the graph,
  and the narrow phase's contact rows are never used by a step whose settings differ from the last solve's (they were
  written with that solve's settings), also when that step captures its graph right after a replay with other settings.
* Contact-free joint worlds (revolute and prismatic springs, limits, motors, distance joints, welds soft and rigid, mouse
  joints, kinematic carriages) at one and eight sub-steps, no relax sweep, dt = 1/30, colour schedule.
* Joint reactions at one and eight sub-steps: impulses times the sub-step rate (the step rate for TGS_Sticky).

Mutations these tests catch: TGS_Soft's contact clamp at a third of the sub-step rate instead of a quarter
(test_reference_order_at_settings at S = 1) and a graph replayed after a solve with other settings without marking its
schedule dirty (test_settings_change_mid_run), neither caught by the tests at (1/60, 4, 2); the body damping formed with dt
instead of the sub-step h in the per-body warm gather (test_first_touch_table_at_settings, test_production_schedule_at_settings
and test_reference_order_at_settings at S > 1); TGS_Soft's first relax-fold segment run S times instead of S - 1; the relax
sweeps of TGS_Soft and SoftStep leaving the warm-start impulses unwritten. Forcing the bias sweep to write them at E > 0
changes no value: the relax sweep of the same sub-step rewrites every contact's warm-start impulses before the next
sub-step's warm start reads them."""
import numpy as np
import pytest

import joint_oracle
from solver2d_b200 import capi, device, scenes
from test_distance_gpu import _distance_world, _step_and_compare
from test_e2e_gpu import _angles, _positions, _ref_pair_table
from test_multistep_gpu import _run
from test_oracle_cpu import VARIANTS
from test_regions_gpu import piles
from test_soft_weld_gpu import _soft_weld_world
from test_spring_gpu import _spring_world
from test_step_settings_cpu import SETTING_IDS, SETTINGS

pytestmark = pytest.mark.gpu
DT = 1.0 / 60.0
# variants whose program prepares its contacts in a pass the narrow phase can take over (COP_PREPARE / COP_PREPARE_COLD)
ROWS_FROM_NARROWPHASE = {"Jacobi", "PGS", "PGS_NGS", "PGS_Soft", "SoftStep", "TGS_Soft", "TGS_NGS", "XPBD"}


@pytest.fixture(scope="module")
def product():
    return capi.Solver2D(device.LIB_PATH)


def _steps(solver, steps):
    """Jacobi blows scenes apart in the reference as well: a few steps show it, more only measure the explosion."""
    return min(steps, 8) if solver == "Jacobi" else steps


# ---- (a) the reference's own order ---------------------------------------------------------------------------------------

@pytest.mark.parametrize("setting", SETTINGS, ids=SETTING_IDS)
@pytest.mark.parametrize("solver", VARIANTS)
def test_reference_order_at_settings(reference, product, dev, solver, setting):
    """scenes.damped_mix with its damped revolute chain: the reference running free, the device in its order."""
    R, P = reference, product
    dt, S, E, warm = setting
    sr = scenes.damped_mix(R, solver, joints=True)
    sp = scenes.damped_mix(P, solver, joints=True)
    dw = device.DeviceWorld.attach(dev, sp.world)
    dw.set_schedule(device.SCHEDULE_WAVEFRONT)
    contacts = 0
    try:
        for step in range(_steps(solver, 24)):
            R.step_collide(sr.world)
            keys, *_ = _ref_pair_table(R, sr.world)
            dw.set_contact_order(keys)
            R.step_solve(sr.world, dt, S, E, warm)
            R.step_finalize(sr.world)
            sp.step(dt, S, E, warm)
            assert np.array_equal(_positions(R, sr), _positions(P, sp)), f"{solver} step {step}: positions"
            assert np.array_equal(_angles(R, sr), _angles(P, sp)), f"{solver} step {step}: angles"
            contacts += dw.counters().constraintCount
        assert contacts > 0
    finally:
        sr.destroy()
        sp.destroy()


# ---- (b) the production schedule at each setting --------------------------------------------------------------------------

def _counting(seen):
    def after(dw):
        seen.append(dw.counters())
    return after


def _pyramid(lib, solver):
    return scenes.pyramid(lib, solver, base_count=10)


def _damped(lib, solver):
    return scenes.damped_mix(lib, solver)


PRODUCTION_SCENES = {"pyramid": _pyramid, "damped_mix": _damped, "limited_chains": scenes.limited_chains}


@pytest.mark.parametrize("setting", SETTINGS, ids=SETTING_IDS)
@pytest.mark.parametrize("scene", sorted(PRODUCTION_SCENES))
@pytest.mark.parametrize("solver", VARIANTS)
def test_production_schedule_at_settings(reference, product, dev, solver, scene, setting):
    seen = []
    _run(reference, product, dev, PRODUCTION_SCENES[scene], solver, _steps(solver, 10), 0, 0, {},
         after_step=_counting(seen), settings=lambda step: setting)
    last = seen[-1]
    if solver != "Jacobi":  # Jacobi's pile is apart within a few steps
        assert max(c.constraintCount for c in seen) > 0
    if scene == "pyramid" and solver != "Jacobi":
        # a pile that stands still: the stage is replayed as a graph, and the narrow phase writes the contact rows
        assert last.graphReplays > 0
        if solver in ROWS_FROM_NARROWPHASE:
            assert last.narrowphaseRowSteps > 0


@pytest.mark.parametrize("setting", SETTINGS, ids=SETTING_IDS)
def test_first_touch_table_at_settings(reference, product, dev, setting):
    """TGS_Soft on scenes.damped_mix (no joints, no kinematic bodies) with the region-local schedule off: the bias sweep
    warm-starts each block's first-touched bodies from the table built with the schedule (s2bFirstTableHeaderKernel), and
    damps them there, whenever warm starting is on. The default mode takes regions on this scene, which skip the table."""
    seen = []
    _run(reference, product, dev, _damped, "TGS_Soft", 10, 0, 0, {}, setup=lambda dw: dw.set_regions(0),
         after_step=_counting(seen), settings=lambda step: setting)
    if setting[3]:
        assert max(c.firstTable for c in seen) > 0
    else:
        assert max(c.firstTable for c in seen) == 0


@pytest.mark.parametrize("setting", SETTINGS, ids=SETTING_IDS)
def test_resident_regions_at_settings(reference, product, dev, setting):
    """TGS_Soft, two piles of 300 boxes, region-local schedule forced: the regions keep their bodies in shared memory
    whenever warm starting is on."""
    seen = []
    _run(reference, product, dev, piles([300, 300]), "TGS_Soft", 6, 0, 0, {}, setup=lambda dw: dw.set_regions(2),
         after_step=_counting(seen), settings=lambda step: setting)
    assert all(c.regionCount > 0 for c in seen)
    assert [c.residentRegions for c in seen] == [1 if setting[3] else 0] * len(seen)


# ---- (c) settings that change between steps -------------------------------------------------------------------------------

A = (DT, 4, 2, True)
B = (1.0 / 30.0, 2, 3, True)
PAUSED = (0.0, 4, 2, True)
COLD = (DT, 4, 2, False)


def _sequence(name, n):
    """The settings of each step; `n`: the length of a run of equal steps."""
    if name == "A-B-A":
        return [A] * n + [B] * n + [A] * n
    if name == "alternating":  # A's graph is replayed after B's eager solve, then B's captured after A's replay
        return [A] * n + [B, A] * n
    if name == "warm_start_alternating":  # the same with warm starting off and on: the schedules and rows differ
        return [A] * n + [COLD, A] * n
    if name == "paused":
        return [A] * n + [PAUSED] * 3 + [A] * n
    if name == "warm_start_off_then_on":
        return [COLD] * 4 + [A] * n
    if name == "substeps_4_1_8":
        return [A] * n + [(DT, 1, 2, True)] * n + [(DT, 8, 2, True)] * n
    if name == "relax_2_0_2":
        return [A] * n + [(DT, 4, 0, True)] * n + [A] * n
    raise KeyError(name)


SEQUENCES = ["A-B-A", "alternating", "warm_start_alternating", "paused", "warm_start_off_then_on", "substeps_4_1_8", "relax_2_0_2"]


@pytest.mark.parametrize("sequence", SEQUENCES)
@pytest.mark.parametrize("solver", VARIANTS)
def test_settings_change_mid_run(reference, product, dev, solver, sequence):
    steps = _sequence(sequence, 3 if solver == "Jacobi" else 6)
    seen = []
    base = {}
    _run(reference, product, dev, _pyramid, solver, len(steps), 0, 0, {},
         setup=lambda dw: base.setdefault("c", dw.counters()), after_step=_counting(seen), settings=lambda step: steps[step])
    replays = [base["c"].graphReplays] + [c.graphReplays for c in seen]
    rows = [base["c"].narrowphaseRowSteps] + [c.narrowphaseRowSteps for c in seen]
    solved = None  # the settings of the last step that ran the solver stage (XPBD skips it on a paused step)
    for k, setting in enumerate(steps):
        # the narrow phase writes a step's contact rows with the last solve's settings: a step with other settings, replayed
        # or captured, marks its schedule dirty and prepares its contacts itself
        if solved is not None and setting != solved:
            assert rows[k + 1] == rows[k], f"step {k}: the narrow phase's rows, written with other settings, were used"
        if not (solver == "XPBD" and setting[0] == 0.0):
            solved = setting
    stable_rows = 0
    k = 0
    while k < len(steps):
        end = k
        while end + 1 < len(steps) and steps[end + 1] == steps[k]:
            end += 1
        # steps k..end share their settings
        # (XPBD skips a paused step's solver stage altogether, reference src/solve_xpbd.c:345-353)
        if end - k + 1 >= 3 and solver != "Jacobi" and not (solver == "XPBD" and steps[k][0] == 0.0):
            assert replays[end + 1] > replays[k + 1], f"steps {k}..{end}: no graph replay"
            stable_rows += rows[end + 1] - rows[k + 1]
        k = end + 1
    if solver in ROWS_FROM_NARROWPHASE and solver != "Jacobi":
        assert stable_rows > 0, "the narrow phase never wrote the contact rows within a run of equal steps"


# ---- (d) contact-free joint worlds ----------------------------------------------------------------------------------------

JOINT_WORLDS = {"springs": _spring_world, "distance": _distance_world, "soft_welds": _soft_weld_world}


@pytest.mark.parametrize("substeps", [1, 8])
@pytest.mark.parametrize("world", sorted(JOINT_WORLDS))
@pytest.mark.parametrize("solver", VARIANTS)
def test_joint_worlds_at_substeps(product, dev, solver, world, substeps):
    P = product
    build = JOINT_WORLDS[world]
    wid, _, _ = build(P, solver)
    P.s2World_Step(wid, 1.0 / 30.0, substeps, 0, True)  # uploads the world
    dw = device.DeviceWorld.attach(dev, wid)
    dw.set_schedule(device.SCHEDULE_COLOR)
    _step_and_compare(P, wid, dw, joint_oracle.load(), solver, 30, colour=True, dt=1.0 / 30.0, substeps=substeps, relax=0)
    P.s2DestroyWorld(wid)


# ---- (e) reactions --------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("substeps", [1, 8])
@pytest.mark.parametrize("solver", ["TGS_Soft", "PGS", "TGS_NGS", "TGS_Sticky", "PGS_NGS_Block"])
def test_reactions_at_substeps(product, dev, solver, substeps):
    """s2Joint_GetReactionForce / GetReactionTorque equal s2ComputeJointReaction on the downloaded rows at the context's
    inv_h (substeps / dt for the sub-stepping variants, 1 / dt for the others), except for TGS_Sticky at inv_dt."""
    P = product
    wid, joints, _ = _soft_weld_world(P, solver)
    for _ in range(20):
        P.s2World_Step(wid, DT, substeps, 1, True)
    ctx = device.make_context(solver, DT, substeps, 1, True)
    rate = np.float32(ctx.inv_dt if solver == "TGS_Sticky" else ctx.inv_h)
    dw = device.DeviceWorld.attach(dev, wid)
    rows = dw.download_joints()
    bodies = dw.download_all_bodies()
    loaded = 0
    for j in joints:
        r = rows[j.index]
        q = bodies["rot"][int(r["bodyA"])]
        x = P.s2ComputeJointReaction((int(r["flags"]) >> 1) & 7, capi.Vec2(*r["impulse"]), float(r["motorImpulse"]),
                                     float(r["lowerImpulse"]), float(r["upperImpulse"]), capi.Rot(float(q[0]), float(q[1])),
                                     capi.Vec2(*r["localAxisA"]), float(rate))
        f, t = P.s2Joint_GetReactionForce(j), P.s2Joint_GetReactionTorque(j)
        assert (np.float32(f.x), np.float32(f.y), np.float32(t)) == (np.float32(x.force.x), np.float32(x.force.y),
                                                                     np.float32(x.torque))
        loaded += int(abs(f.x) + abs(f.y) + abs(t) > 0.0)
    assert loaded >= 7
    P.s2DestroyWorld(wid)
