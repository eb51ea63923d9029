"""CPU: bullets (s2Body_SetBullet, DESIGN.md §3.12) without a device.

* The bullets scene builds and steps on the reference, which has no bullets: projectiles tunnel through their targets
  there, and the calls appear in `lib.missing`.
* The host restatement of the bullet pass (`host_bullet_pass`, which the GPU tests compare the device against bit for
  bit) is checked on hand-built rows: its candidate rule (static, kinematic and non-bullet dynamic shapes; not the
  bullet's own body, not other bullets, not filtered or jointed pairs, no segment pair) and its earliest fraction, against
  the float64 sweep of test_toi_reference_cpu."""
import ctypes as C

import numpy as np
import pytest

from solver2d_b200 import capi, device, scenes
from test_continuous_gpu import _core_approaches, _fast, _sweep
from test_toi_reference_cpu import TARGET, TOL, Shape64, Sweep64, min_sep64, sep64

BULLET = 0x20  # S2B_BODY_BULLET


@pytest.fixture(scope="module")
def lib():
    return capi.Solver2D(device.LIB_PATH)


def _should_collide(fa, fb):
    """s2bShouldShapesCollide: (category, mask, group) per shape."""
    if fa[2] == fb[2] and fa[2] != 0:
        return fa[2] > 0
    return (fa[1] & fb[0]) != 0 and (fa[0] & fb[1]) != 0


def _is_bullet(row):
    f = int(row["flags"])
    return (f & 1) != 0 and ((f >> 1) & 3) == 2 and (f & BULLET) != 0


def _still(row):
    return capi.Sweep(capi.Vec2(*row["localCenter"]), capi.Vec2(*row["position"]), capi.Vec2(*row["position"]),
                      capi.Rot(*row["rot"]), capi.Rot(*row["rot"]))


def host_bullet_pass(P, shapes, before, after, joints=frozenset(), reach=8.0):
    """The bullet pass restated on the host: body slot -> (fraction, sweep) for every bullet it clamps.

    `shapes`: per shape a dict with `body` (slot), `form` (capi.Polygon in the body frame), `filter` ((category, mask,
    group)) and `segment` (a segment shape: no core, and no manifold with another segment). `before` / `after`: body rows
    at the start of the step and before the bullet pass (the final poses of every other body). `joints`: jointed body
    pairs (sorted tuples). Shapes beyond `reach` metres of a bullet's start are skipped (a prefilter: the scenes keep every
    candidate well inside it)."""
    out = {}
    for b in range(len(after)):
        if not _is_bullet(after[b]) or not _fast(before[b], after[b]):
            continue
        sweep = _sweep(before[b], after[b])
        earliest = 1.0
        for s in (s for s in shapes if s["body"] == b):
            form = s["form"]
            ext = P.s2ComputeShapeExtent(C.byref(form), capi.Vec2(*before[b]["localCenter"]))
            pb = P.s2MakeProxy(form.vertices, form.count, form.radius)
            for o in shapes:
                ob = o["body"]
                if ob == b or _is_bullet(after[ob]) or int(after[ob]["flags"]) & 1 == 0:
                    continue
                if not _should_collide(s["filter"], o["filter"]) or tuple(sorted((b, ob))) in joints:
                    continue
                if s["segment"] and o["segment"]:
                    continue
                if np.hypot(*(np.array(after[ob]["position"]) - np.array(before[b]["position"]))) > reach:
                    continue
                ws = _still(after[ob])
                of = o["form"]
                pa = P.s2MakeProxy(of.vertices, of.count, of.radius)
                res = P.s2TimeOfImpact(C.byref(capi.TOIInput(pa, pb, ws, sweep, 1.0)))
                if res.state == capi.TOI_OVERLAPPED and ext.minExtent <= 0.0:
                    continue  # a segment has no core: touching at the start, it is let go
                if res.state == capi.TOI_OVERLAPPED:
                    core = (capi.Vec2 * 1)(ext.center)
                    pc = P.s2MakeProxy(core, 1, np.float32(0.25) * np.float32(ext.minExtent))
                    res = P.s2TimeOfImpact(C.byref(capi.TOIInput(pa, pc, ws, sweep, 1.0)))
                    if res.state == capi.TOI_OVERLAPPED and _core_approaches(P, pa, ws, core, sweep):
                        earliest = 0.0
                        continue
                if res.state in (capi.TOI_HIT, capi.TOI_FAILED):
                    earliest = min(earliest, res.fraction)
        if earliest < 1.0:
            out[b] = (earliest, sweep)
    return out


def test_reference_has_no_bullets_and_tunnels(reference):
    assert "s2Body_SetBullet" in reference.missing and "s2Body_IsBullet" in reference.missing
    sc = scenes.bullets(reference, "TGS_Soft")
    lanes = sc.piles["lanes"]
    ever = np.zeros(len(lanes), dtype=bool)
    for _ in range(30):
        sc.step(1.0 / 60.0, 4, 2, True)
        ever |= scenes.bullets_behind(reference, sc)
    meant = np.array([lane["passes"] for lane in lanes])
    assert ever[meant].all()
    assert ever[~meant].sum() >= 1
    assert {lane["kind"] for lane, e in zip(lanes, ever) if e and not lane["passes"]} == set(scenes.BULLET_TARGETS)
    sc.destroy()


# ---- the restatement on hand-built rows ---------------------------------------------------------------------------

def _row(rows, i, kind, pos, rot=(0.0, 1.0), flags_extra=0, lc=(0.0, 0.0), ext=(0.1, 0.1)):
    r = rows[i]
    r["index"] = i
    r["flags"] = 1 | (kind << 1) | flags_extra
    r["position"] = pos
    r["origin"] = (pos[0] - lc[0], pos[1] - lc[1])
    r["rot"] = rot
    r["localCenter"] = lc
    r["minExtent"], r["maxExtent"] = ext


def _box(lib, hx, hy):
    return lib.s2MakeBox(hx, hy)


def _circle(r):
    p = capi.Polygon()
    p.count, p.radius = 1, r
    return p


def _poly64(form):
    return Shape64([(form.vertices[k].x, form.vertices[k].y) for k in range(form.count)], form.radius)


def _sweep64(row0, row1):
    return Sweep64(row0["localCenter"], row0["position"], row1["position"], row0["rot"], row1["rot"])


def _lane(lib, kind, x, flags_extra=0, filt=(1, 0xFFFFFFFF, 0), form=None, segment=False):
    return dict(kind=kind, x=x, flags_extra=flags_extra, filter=filt, form=form or _box(lib, 0.025, 1.0), segment=segment)


def _hand_world(lib, targets, bullet_filter=(1, 0xFFFFFFFF, 0)):
    """A 0.1 m circle bullet at slot 0 moving from x = 0 to x = 4 in one step, and one target per entry of `targets` at
    slots 1.., each still at its x. Returns (shapes, before, after)."""
    n = 1 + len(targets)
    before = np.zeros(n, dtype=device.BODY_ROW)
    after = np.zeros(n, dtype=device.BODY_ROW)
    _row(before, 0, 2, (0.0, 0.0), flags_extra=BULLET)
    _row(after, 0, 2, (4.0, 0.0), flags_extra=BULLET)
    shapes = [dict(body=0, form=_circle(0.1), filter=bullet_filter, segment=False)]
    for k, t in enumerate(targets, start=1):
        for rows in (before, after):
            _row(rows, k, t["kind"], (t["x"], 0.0), flags_extra=t["flags_extra"])
        shapes.append(dict(body=k, form=t["form"], filter=t["filter"], segment=t["segment"]))
    return shapes, before, after


@pytest.mark.parametrize("first", ["static", "kinematic", "dynamic", "bullet", "filtered", "jointed", "own"])
def test_candidate_rule_and_earliest_against_float64(lib, first):
    """The first thing in the bullet's path is `first`; a dynamic plank lies behind it. The pass must stop the bullet at
    `first` when the rules make it a candidate, and at the plank behind it when they do not."""
    kinds = {"static": 0, "kinematic": 1, "dynamic": 2, "bullet": 2, "filtered": 2, "jointed": 2}
    behind = _lane(lib, 2, 3.0)
    joints = frozenset()
    if first == "own":
        shapes, before, after = _hand_world(lib, [behind])
        # a second shape of the bullet's own body, ahead of it: never a candidate
        shapes.append(dict(body=0, form=_box(lib, 0.025, 1.0), filter=(1, 0xFFFFFFFF, 0), segment=False))
        held = False
    else:
        extra = BULLET if first == "bullet" else 0
        filt = (2, 0xFFFFFFFF, 0) if first == "filtered" else (1, 0xFFFFFFFF, 0)
        shapes, before, after = _hand_world(lib, [_lane(lib, kinds[first], 1.5, extra, filt), behind],
                                            bullet_filter=(1, 0xFFFFFFFF & ~2, 0))
        if first == "jointed":
            joints = frozenset({(0, 1)})
        held = first in ("static", "kinematic", "dynamic")
    got = host_bullet_pass(lib, shapes, before, after, joints)
    assert list(got) == [0]
    t, _ = got[0]
    stop = 1 if held else len(after) - 1
    A = _poly64(shapes[0]["form"])
    sw = _sweep64(before[0], after[0])
    for k, s in enumerate(shapes[1:], start=1):
        if s["body"] != stop:
            continue
        o = _poly64(s["form"])
        still = _sweep64(after[s["body"]], after[s["body"]])
        # at the fraction: at the target separation within the tolerance; before it: never closer
        d = float(sep64(o, still, A, sw, [t])[0])
        assert TARGET - TOL - 1e-5 <= d <= TARGET + TOL + 1e-5, (first, t, d)
        lo, _ = min_sep64(o, still, A, sw, 0.0, t)
        assert lo >= TARGET - TOL - 1e-5, (first, lo)
    # the nearer thing it was let through lies behind the bullet's centre at the fraction taken (the centre moves 4 m)
    if not held:
        assert 4.0 * t > 1.5, (first, t)


def test_segment_pairs_and_starting_contact(lib):
    """A segment-carrying bullet never collides with a segment target; a bullet that starts touching a target and moves
    away from it is let go, one that starts touching and moves into it is held at 0."""
    seg = lib.s2MakeCapsule(capi.Vec2(0.0, -1.0), capi.Vec2(0.0, 1.0), 0.0)
    shapes, before, after = _hand_world(lib, [_lane(lib, 0, 1.5, form=seg, segment=True)])
    shapes[0] = dict(body=0, form=lib.s2MakeCapsule(capi.Vec2(0.0, -0.1), capi.Vec2(0.0, 0.1), 0.0), filter=(1, 0xFFFFFFFF, 0),
                     segment=True)
    assert host_bullet_pass(lib, shapes, before, after) == {}
    # starting within the target of a box just behind the start, moving away: let go
    shapes, before, after = _hand_world(lib, [_lane(lib, 2, -0.126)])
    assert host_bullet_pass(lib, shapes, before, after) == {}
    # starting deep in a box ahead (the core within the target too) and moving into it: held at its start
    # (the core, of radius 0.025, 0.003 m from the box's face)
    shapes, before, after = _hand_world(lib, [_lane(lib, 2, 0.078, form=_box(lib, 0.05, 1.0))])
    got = host_bullet_pass(lib, shapes, before, after)
    assert list(got) == [0] and got[0][0] == 0.0
