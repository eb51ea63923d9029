"""GPU: the solver's hub-body paths on both sides of their capacity limits, against the oracle replayed in the device's
solve order, tolerance 0. A hub is a body with more than 48 incident constraints (a container wall, a tray under a pile);
its constraints take the serial overflow group, its incidence list a block-wide sort, its warm start a block-wide gather.
Each of those has a fast form of fixed size and a fallback; the scenes (tests/hub_cases.py, their sizes checked on the
reference's own tables by tests/test_hub_capacity_cpu.py) sit on either side of every limit:

1. the serial group staged in shared memory (persistent.cuh, S2B_OV_MAX_*): 1024 / 1025 distinct bodies, 2048 / 2049
   contacts, 256 / 257 joints as revolute (limits and motor on), weld, prismatic and motor rows, with a mouse joint on the
   hub. All ten variants, persistent kernel on and off, regions 0 and 2.
2. incidence lists of 8, 9-24, 24 / 25, 33, 512 / 513, 1025, 2048 / 2049 and 3000 entries (register sort, insertion sort,
   bitonic sort padded to a power of two, heap sort). All ten variants, persistent kernel on and off, regions 0 and 2;
   the ticketed passes that read the lists' ordinals on 2048 / 2049 / 3000, all ten variants.
3. the block-wide warm-start gather over lists of 513 to 3000 entries (more than one 512-thread chunk), gather on and off,
   and 540 hubs, more than the persistent grid has blocks (at most 4 x SM count), so blocks loop over hubs. The five
   sub-stepping variants (the gather serves only them), regions 0 and 2.
4. the colour limit: S2B_HUB_DEGREE=0 and 64 colours on a hub of 100 constraints: 64 colours, 36 overflow. With regions
   (mode 2) the hub belongs to no region, so its constraints are the cut set and colour 63 takes the largest cut key, the
   last device-wide group before the serial one. All ten variants, persistent kernel on and off, regions 0 and 2.
5. the colouring threshold (S2B_HUB_DEGREE) against the fixed S2B_HEAVY_DEGREE of the regions and the gather: degree 60
   under 100, degree 40 under 30, and degrees 48 and 49 at the defaults. All ten variants, persistent kernel on and off,
   regions 0 and 2.

Every case asserts the size it reached (serial group, list lengths, hub count, colours), computed from the rows and the
solve order the device reports, so that a scene that drifts off its edge fails instead of passing on the other side.
Contacts and joints are warm-started with seeded random impulses: a gather that sums in a wrong order or skips a chunk
then changes bits."""
import numpy as np
import pytest
import torch

import hub_cases
import joint_oracle
from helpers import bit_equal
from hub_cases import SCENES, build_rows, check_sizes, degrees, item_ends
from oracle import port
from solver2d_b200 import capi, device

pytestmark = pytest.mark.gpu
DT = hub_cases.DT
VARIANTS = ["Jacobi", "PGS", "PGS_NGS", "PGS_NGS_Block", "PGS_Soft", "SoftStep", "TGS_Sticky", "TGS_Soft", "TGS_NGS", "XPBD"]
SUBSTEPPING = ["SoftStep", "TGS_Sticky", "TGS_Soft", "TGS_NGS", "XPBD"]

_rows = {}


def _scene_rows(reference, name, solver):
    key = (name, solver)
    if key not in _rows:
        b, c, j, sc = build_rows(reference, name, solver)
        _rows[key] = (b, c, j, [sc.joints[k].index for k in sc.piles.get("pendulum", [])])
    b, c, j, pend = _rows[key]
    return b.copy(), c.copy(), j.copy(), pend


def _convert(joints, slots, kind):
    """Turn the beam's stand-in revolute pendulum rows into rows of joint type `kind`."""
    if kind in ("revolute", None):
        return joints
    s = np.asarray(slots, dtype=np.int64)
    assert np.all((joints["flags"][s] & (device.JOINT_ENABLE_LIMIT | device.JOINT_ENABLE_MOTOR)) == 0)
    base = joints["flags"][s] & ~0xE
    if kind == "weld":
        joints["flags"][s] = base | (device.JOINT_WELD << 1)
    elif kind == "prismatic":
        joints["flags"][s] = base | (device.JOINT_PRISMATIC << 1) | device.JOINT_ENABLE_LIMIT | device.JOINT_ENABLE_MOTOR
        joints["lowerAngle"][s] = -0.05
        joints["upperAngle"][s] = 0.05
        joints["maxMotorTorque"][s] = 3.0
        joints["motorSpeed"][s] = np.where(s % 2 == 0, 0.4, -0.2).astype(np.float32)
        joints["referenceAngle"][s] = 0.0
        joints["localAxisA"][s] = (0.0, 1.0)
    elif kind == "motor":
        joints["flags"][s] = base | (device.JOINT_MOTOR << 1)
        joints["localOriginAnchorB"][s] = (0.0, 0.0)
        joints["referenceAngle"][s] = 0.1
        joints["maxMotorTorque"][s] = 2.0
        joints["motorSpeed"][s] = 0.0
        joints["hertz"][s] = 20.0
        joints["dampingRatio"][s] = 0.3
    return joints




def _run(reference, dev, monkeypatch, name, solver, persistent=True, regions=0, kind=None, gather=True, dataflow=False,
         max_colors=None, hub_degree=None):
    """One solver stage of scene `name` on the device against the oracle in the device's order. Returns (order,
    group_sizes, counters, bodies, contacts, joints)."""
    if hub_degree is not None:
        monkeypatch.setenv("S2B_HUB_DEGREE", str(hub_degree))
    bodies, contacts, joints, pend = _scene_rows(reference, name, solver)
    joints = _convert(joints, pend, kind)
    rng = np.random.default_rng(11)
    for j in range(2):
        has = contacts["pointCount"] > j
        contacts["points"]["normalImpulse"][has, j] = rng.uniform(0.0, 0.05, int(has.sum())).astype(np.float32)
        contacts["points"]["tangentImpulse"][has, j] = rng.uniform(-0.02, 0.02, int(has.sum())).astype(np.float32)
    jv = (joints["flags"] & 1) == 1
    n = int(jv.sum())
    joints["impulse"][jv] = rng.uniform(-0.05, 0.05, (n, 2)).astype(np.float32)
    joints["motorImpulse"][jv] = rng.uniform(-0.02, 0.02, n).astype(np.float32)
    joints["lowerImpulse"][jv] = rng.uniform(0.0, 0.02, n).astype(np.float32)
    joints["upperImpulse"][jv] = rng.uniform(0.0, 0.02, n).astype(np.float32)
    ctx = device.make_context(solver, DT, 4, 2)

    dw = dev.create_world(capi.SOLVER[solver])
    dw.upload_bodies(bodies, len(bodies))
    dw.upload_joints(joints, len(joints))
    dw.upload_contacts(contacts)
    dw.set_schedule(device.SCHEDULE_COLOR)
    dw.set_persistent(persistent)
    dw.set_regions(regions)
    dw.set_warm_gather(gather)
    dw.set_dataflow(dataflow)
    if max_colors is not None:
        dw.set_max_colors(max_colors)
    dw.solve(ctx)
    got = dw.download_all_bodies(len(bodies))
    got_contacts = dw.download_contacts(len(contacts))
    got_joints = dw.download_joints(len(joints))
    order, group_sizes = dw.solve_order(len(contacts) + len(joints))
    counters = dw.counters()
    dw.destroy()
    monkeypatch.delenv("S2B_HUB_DEGREE", raising=False)
    assert len(order) == int((contacts["pointCount"] > 0).sum()) + n

    # within a parallel group no movable body appears twice
    mov = hub_cases.movable(bodies)
    parallel = len(group_sizes) - (1 if counters.overflowCount > 0 else 0)
    group_of = np.repeat(np.arange(len(group_sizes)), group_sizes)
    ea, eb = _ends(order, contacts, joints)
    both = np.concatenate([np.stack([group_of, ea], 1), np.stack([group_of, eb], 1)])
    both = both[(both[:, 1] >= 0) & (both[:, 0] < parallel)]
    both = both[mov[both[:, 1]]]
    _, cnt = np.unique(both[:, 0].astype(np.int64) * (len(bodies) + 1) + both[:, 1], return_counts=True)
    assert (cnt == 1).all(), "a movable body appears twice in a parallel group"

    O = port.load() if kind in (None, "revolute") else joint_oracle.load()
    ob, oc, oj = O.solve(capi.SOLVER[solver], bodies, contacts, joints, ctx, order=order)
    valid = (bodies["flags"] & 1) == 1
    for field in ("position", "rot", "linearVelocity", "angularVelocity"):
        g = np.ascontiguousarray(got[field][valid]).reshape(int(valid.sum()), -1)
        o = np.ascontiguousarray(ob[field][valid]).reshape(int(valid.sum()), -1)
        bad = np.nonzero((g.view(np.uint32) != o.view(np.uint32)).any(axis=1))[0]
        assert len(bad) == 0, f"{name} {solver}: {field} differs at bodies {np.nonzero(valid)[0][bad[:8]].tolist()}"
    live = contacts["pointCount"] > 0
    for field in ("normalImpulse", "tangentImpulse"):
        assert bit_equal(got_contacts["points"][field][live], oc["points"][field][live]), field
    for field in ("impulse", "motorImpulse", "lowerImpulse", "upperImpulse"):
        assert bit_equal(got_joints[field][jv], oj[field][jv]), field
    return order, group_sizes, counters, bodies, contacts, joints


def _ends(order, contacts, joints):
    """Raw body indices of each solved item (a mouse joint: -1 on side A)."""
    is_c = order >= 0
    ci = np.where(is_c, order, 0)
    ji = np.where(is_c, 0, -1 - order)
    mouse = ((joints["flags"][ji] >> 1) & 7) == device.JOINT_MOUSE
    ea = np.where(is_c, contacts["bodyA"][ci] if len(contacts) else -1, np.where(mouse, -1, joints["bodyA"][ji]))
    eb = np.where(is_c, contacts["bodyB"][ci] if len(contacts) else -1, joints["bodyB"][ji])
    return ea.astype(np.int64), eb.astype(np.int64)


def _serial_sizes(order, group_sizes, counters, contacts, joints):
    """(contacts, joints, distinct bodies, movable or not) of the serial group as the device ran it: its last group."""
    if counters.overflowCount == 0:
        return (0, 0, 0)
    items = order[len(order) - group_sizes[-1]:]
    is_c = items >= 0
    ci, ji = items[is_c], -1 - items[~is_c]
    ends = np.concatenate([contacts["bodyA"][ci], contacts["bodyB"][ci], joints["bodyA"][ji], joints["bodyB"][ji]])
    return int(is_c.sum()), int((~is_c).sum()), len(np.unique(ends[ends >= 0]))


# ---- 1. the serial group at each staging limit ---------------------------------------------------------------------------

STAGING = [("bodies_1024", None), ("bodies_1025", None), ("contacts_2048", None), ("contacts_2049", None),
           ("joints_256_limits_motor", "revolute"), ("joints_257_limits_motor", "revolute"), ("joints_256", "weld"),
           ("joints_257", "weld"), ("joints_256", "prismatic"), ("joints_257", "prismatic"), ("joints_256", "motor"),
           ("joints_257", "motor")]


@pytest.mark.parametrize("regions", [0, 2])
@pytest.mark.parametrize("persistent", [True, False])
@pytest.mark.parametrize("solver", VARIANTS)
@pytest.mark.parametrize("name,kind", STAGING)
def test_serial_group_at_staging_limits(reference, dev, monkeypatch, name, kind, solver, persistent, regions):
    order, sizes, c, b, ct, j = _run(reference, dev, monkeypatch, name, solver, persistent, regions, kind=kind)
    want = SCENES[name][1]["serial"]
    got = _serial_sizes(order, sizes, c, ct, j)
    assert got == want
    # the side of the staging limits the device's serial group fell on is the one the scene is named for
    staged = got[0] <= hub_cases.OV_MAX_CONTACTS and got[1] <= hub_cases.OV_MAX_JOINTS and got[2] <= hub_cases.OV_MAX_BODIES
    assert staged == name.endswith(("_1024", "_2048", "_256", "_256_limits_motor"))
    check_sizes(name, b, ct, j)


# ---- 2. incidence-list lengths on every side of the sorts -----------------------------------------------------------------

@pytest.mark.parametrize("regions", [0, 2])
@pytest.mark.parametrize("persistent", [True, False])
@pytest.mark.parametrize("solver", VARIANTS)
def test_incidence_list_lengths(reference, dev, monkeypatch, solver, persistent, regions):
    order, sizes, c, b, ct, j = _run(reference, dev, monkeypatch, "lists", solver, persistent, regions)
    deg = check_sizes("lists", b, ct, j)
    for n in (8, 9, 12, 16, 24, 25, 33, 512, 513, 1025, 3000):
        assert (deg == n).any(), n
    assert deg.max() > hub_cases.LONG_LIST_SHARED and ((deg > hub_cases.LONG_LIST) & (deg <= 32)).any()


@pytest.mark.parametrize("solver", VARIANTS)
@pytest.mark.parametrize("name", ["contacts_2048", "contacts_2049", "lists"])
def test_ticketed_passes_on_long_lists(reference, dev, monkeypatch, name, solver):
    """The ticketed passes wait on each constraint's ordinal in its bodies' sorted lists (bitonic at 2048, heap sort at
    2049 and 3000)."""
    order, sizes, c, b, ct, j = _run(reference, dev, monkeypatch, name, solver, True, 0, dataflow=True)
    assert max(check_sizes(name, b, ct, j)) in (2048, 2049, 3000)


# ---- 3. the block-wide warm-start gather ----------------------------------------------------------------------------------

@pytest.mark.parametrize("gather", [True, False])
@pytest.mark.parametrize("regions", [0, 2])
@pytest.mark.parametrize("solver", SUBSTEPPING)
@pytest.mark.parametrize("name", ["lists", "many_hubs"])
def test_block_gather(reference, dev, monkeypatch, name, solver, regions, gather):
    order, sizes, c, b, ct, j = _run(reference, dev, monkeypatch, name, solver, True, regions, gather=gather)
    hubs = hub_cases.hub_lists(b, ct, j)
    if name == "lists":
        assert [h for h in hubs if h > 512] == [513, 1025, 3000]  # one, two and six 512-thread chunks
    else:
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        assert len(hubs) == 540 and len(hubs) > 4 * sms


# ---- 4. the colour limit --------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("regions", [0, 2])
@pytest.mark.parametrize("persistent", [True, False])
@pytest.mark.parametrize("solver", VARIANTS)
def test_colour_limit(reference, dev, monkeypatch, solver, persistent, regions):
    order, sizes, c, b, ct, j = _run(reference, dev, monkeypatch, "colour_limit", solver, persistent, regions, max_colors=64,
                                     hub_degree=0)
    tray = int(np.argmax(degrees(b, ct, j)))
    ea, eb = _ends(order, ct, j)
    on_tray = (ea == tray) | (eb == tray)
    assert c.overflowCount > 0 and sizes[-1] == 36 and on_tray[len(order) - 36:].all()
    # the other 64 take one group each, the last of them (colour 63) right before the serial group: with regions on, the
    # cut colours' device-wide groups come after every region's groups, so colour 63 holds the largest cut key
    group_of = np.repeat(np.arange(len(sizes)), sizes)
    coloured = group_of[on_tray][:-36]
    assert len(coloured) == 64 and len(set(coloured.tolist())) == 64 and coloured.max() == len(sizes) - 2
    assert np.array_equal(coloured, np.arange(len(sizes) - 65, len(sizes) - 1))
    if regions == 0 or not persistent:
        assert c.regionCount == 0 and len(sizes) == 64 + 1  # colours 0-63, then the serial group
    else:
        assert c.regionCount > 0 and c.cutGroupCount == 64


# ---- 5. thresholds that disagree ------------------------------------------------------------------------------------------

THRESHOLDS = [("degree_60", 100, 64, 60), ("degree_40", 30, None, 20), ("degree_48_49", None, None, 24)]


@pytest.mark.parametrize("regions", [0, 2])
@pytest.mark.parametrize("persistent", [True, False])
@pytest.mark.parametrize("solver", VARIANTS)
@pytest.mark.parametrize("name,hub_degree,max_colors,colours", THRESHOLDS)
def test_thresholds(reference, dev, monkeypatch, name, hub_degree, max_colors, colours, solver, persistent, regions):
    """degree_60: coloured under S2B_HUB_DEGREE=100 (60 colours), yet a hub of the regions and the gather; degree_40: serial
    under S2B_HUB_DEGREE=30, yet no hub; degree_48_49: 48 is coloured (24 colours, the rest serial), 49 goes serial whole."""
    order, sizes, c, b, ct, j = _run(reference, dev, monkeypatch, name, solver, persistent, regions, max_colors=max_colors,
                                     hub_degree=hub_degree)
    check_sizes(name, b, ct, j)
    want = hub_cases.serial_sizes(b, ct, j, hub_degree=hub_degree if hub_degree is not None else hub_cases.HUB_DEGREE)
    serial = _serial_sizes(order, sizes, c, ct, j)
    if name == "degree_48_49":
        want = (want[0] + 24, 0, want[2] + 1)  # the 48-body's 24 constraints beyond 24 colours join the serial group
    assert serial == want
    # the most-coloured body's constraints outside the serial group: one per colour, in either mode
    deg = degrees(b, ct, j)
    body = {"degree_60": 60, "degree_40": 20, "degree_48_49": 48}[name]
    body = int(np.nonzero(deg == body)[0][0])
    ea, eb = _ends(order, ct, j)
    parallel = len(order) - (sizes[-1] if c.overflowCount > 0 else 0)
    assert int(((ea[:parallel] == body) | (eb[:parallel] == body)).sum()) == colours
    if regions == 0:
        assert len(sizes) - (1 if c.overflowCount > 0 else 0) == colours
