"""CPU: the scenes of tests/test_pair_edges_gpu.py run on the reference alone (tests/pair_edges.py).

* Every step, pair_edges.brute_pairs over the reference's own fat boxes equals the reference's contact table: the
  brute-force restatement the GPU tests check the device against is tied to the reference first.
* Every scene reaches the edge it is built for, measured on the reference's data: a scene that drifts off its edge fails
  here, without a GPU."""
import numpy as np
import pytest

import pair_edges as pe
from oracle import ref as refmod
from solver2d_b200 import capi


def _walk(R, name):
    """Run scene `name` on the reference as _run steps it (collide, solve, finalize); per step after the collide:
    (pair keys, fat boxes, body slot by shape slot, body types, shape capacity before the step's pass)."""
    builder, steps = pe.SCENES[name]
    sc = builder(R, "TGS_Soft")
    hook = pe.before_step_for(name)
    out = []
    I = refmod.SHAPE_I
    for step in range(steps):
        if hook is not None:
            hook(step, ((R, sc),))
        cap = R.capacities(sc.world)["shapeCap"]
        R.step_collide(sc.world)
        want, got = pe.ref_pairs(R, sc.world)
        assert want == got, f"{name} step {step}: brute force {len(want)} pairs, reference {len(got)}: " \
                            f"missing {sorted(got - want)[:5]}, extra {sorted(want - got)[:5]}"
        sf, si = R.shapes(sc.world)
        _, bi = R.bodies(sc.world)
        body = np.where(si[:, I["valid"]] == 1, si[:, I["body"]], -1)
        out.append(dict(pairs=got, fat=sf[:, 4:8].copy(), body=body, btype=bi[:, refmod.BODY_I["type"]], cap=cap))
        R.step_solve(sc.world, pe.DT, 4, 2, True)
        R.step_finalize(sc.world)
    sc.destroy()
    return out


@pytest.mark.parametrize("name", sorted(pe.SCENES))
def test_brute_force_equals_reference_every_step(reference, name):
    _walk(reference, name)


def _new_pairs(seen):
    prev, out = set(), []
    for s in seen:
        out.append(len(s["pairs"] - prev))
        prev = s["pairs"]
    return out


def test_lattice_burst_overflows_the_default_pair_buffer(reference):
    """The default buffer is sized on the first pass (8 per shape slot + 1024) and kept: the lattice's new pairs exceed it."""
    seen = _walk(reference, "lattice_burst")
    new = _new_pairs(seen)
    first_cap = seen[0]["cap"]
    assert max(new[:pe.LATTICE_STEP]) <= 8 * first_cap + 1024
    assert new[pe.LATTICE_STEP] > 8 * first_cap + 1024, (new, first_cap)
    assert seen[pe.LATTICE_STEP]["cap"] > first_cap  # the shape pool grew


def test_interleaving_clouds_burst_past_the_small_buffer(reference):
    """No pass before the burst finds more than S2B_PAIR_BUFFER new pairs; the burst, on a step after a pass (so its
    search is the one started behind the step before), does."""
    new = _new_pairs(_walk(reference, "interleaving_clouds"))
    burst = next(k for k, n in enumerate(new) if n > pe.CLOUD_BUFFER)
    assert burst >= 1 and max(new[:burst]) <= pe.CLOUD_BUFFER, new


def _first_pass_large(seen):
    s = seen[0]
    moved = (s["body"] >= 0) & (s["btype"][np.maximum(s["body"], 0)] != capi.STATIC_BODY)  # every new movable proxy
    return pe.large_movers(s["fat"], s["body"], moved)


def _large_by_root(seen):
    """Per pass k >= 1: (large movers under the pass's own root box, under the previous pass's root box). The moved
    proxies of pass k are the shapes whose fat box finalize changed in between."""
    out = []
    for prev, cur in zip(seen, seen[1:]):
        moved = (cur["body"] >= 0) & np.any(prev["fat"] != cur["fat"], axis=1)
        out.append((pe.large_movers(cur["fat"], cur["body"], moved),
                    pe.large_movers(cur["fat"], cur["body"], moved, pe.root_box(prev["fat"], prev["body"]))))
    return out


@pytest.mark.parametrize("name,large", [("large_glide64", 64), ("large_glide65", 65)])
def test_large_glide_counts_every_pass(reference, name, large):
    """Every pass has exactly `large` large movers, under either root box."""
    seen = _walk(reference, name)
    assert _first_pass_large(seen) == large
    assert _large_by_root(seen) == [(large, large)] * (len(seen) - 1)


@pytest.mark.parametrize("name,large", [("one_big255", 0), ("one_big256", 1)])
def test_leaf_threshold_counts(reference, name, large):
    seen = _walk(reference, name)
    assert _first_pass_large(seen) == large
    assert int((seen[0]["body"] >= 0).sum()) == int(name[-3:])


def test_root_flip_step(reference):
    """The previous and the current root box classify the slider differently on ROOT_FLIP_STEP, and only there."""
    seen = _walk(reference, "root_flip")
    assert int((seen[0]["body"] >= 0).sum()) >= pe.LARGE_MIN_LEAVES
    by_root = _large_by_root(seen)
    differ = [k + 1 for k, (cur, prev) in enumerate(by_root) if cur != prev]
    assert differ == [pe.ROOT_FLIP_STEP], by_root
    assert by_root[pe.ROOT_FLIP_STEP - 1] == (0, 1)


def test_tree_height_hand_cases():
    """tree_height on codes: distinct codes 0..n-1 for 1, 2, 8, 9 and 17 leaves; all-equal codes (split on the position);
    a geometric chain 2^j - 1 with duplicates below it."""
    for n, h in ((1, 0), (2, 1), (8, 3), (9, 4), (17, 5)):
        assert pe.tree_height(np.arange(n)) == h
        assert pe.tree_height(np.zeros(n)) == h  # ties: a balanced tree over the sorted positions
    # codes 2^j - 1 (j = 1..15): 2^j - 1 differs from every smaller one in bit j - 1, so the splits peel off 32767,
    # 16383, ..., 3 (14 levels) down to the node holding 1 and the zeros; one more split, then the 6 zero codes
    # (position ties) below: 14 + 1 + 3
    chain = [2 ** j - 1 for j in range(1, 16)] + [0] * 6
    assert pe.tree_height(chain[::-1]) == 18
    assert pe.tree_height(chain) == 18  # the leaf order does not change the tree


def test_morton_codes_hand_cases():
    f = np.float32
    # centres on one horizontal line: the y extent is clamped to 1e-6, every y quantises to 0
    fat = np.array([[0, 5, 2, 7], [4, 5, 6, 7], [8, 5, 10, 7]], f)  # centres 1, 5, 9
    assert pe.morton_codes(fat).tolist() == [0, int(pe.expand_bits(16383)), int(pe.expand_bits(32767))]
    # the corner opposite the minimum gets every bit
    fat = np.array([[0, 0, 2, 2], [8, 8, 10, 10]], f)
    assert pe.morton_codes(fat).tolist() == [0, 0x3FFFFFFF]


@pytest.mark.parametrize("scene,height", [("pyramid447", 18), ("tumbler100", 16)])
def test_restated_height_matches_device_fixture(reference, scene, height):
    """The heights test_broadphase_gpu.TREE_HEIGHT_FIXTURE records for the device's first build of these scenes."""
    from solver2d_b200 import scenes
    R = reference
    sc = scenes.pyramid(R, "TGS_Soft", base_count=447) if scene == "pyramid447" else scenes.tumbler(R, "TGS_Soft", grid=100)
    sf, si = R.shapes(sc.world)
    assert pe.restated_height(sf[:, 4:8], si[:, refmod.SHAPE_I["valid"]] == 1) == height
    sc.destroy()


def test_exact_touch_gaps(reference):
    """A's fat box touches B's and D's exactly (gap 0 along x; D also along y) and is one float32 ulp below C's."""
    seen = _walk(reference, "exact_touch")
    s = seen[0]
    fat = s["fat"]
    live = np.nonzero(s["body"] >= 0)[0]
    a, b, c, d = live[1:5]  # the slider is the first shape
    f32 = np.float32
    assert f32(fat[b, 0] - fat[a, 2]) == 0.0 and f32(fat[d, 0] - fat[a, 2]) == 0.0 and f32(fat[d, 1] - fat[a, 3]) == 0.0
    assert fat[c, 1] == np.nextafter(fat[a, 3], f32(1.0))
    for s in seen:
        assert (a, b) in s["pairs"] and (a, d) in s["pairs"] and (a, c) not in s["pairs"]


def test_launched_row_empties_and_refills(reference):
    counts = [len(s["pairs"]) for s in _walk(reference, "launched_row")]
    empty = [k for k, n in enumerate(counts) if n == 0]
    assert counts[0] == 16 and empty and empty[0] > pe.LAUNCH_STEP and counts[-1] == 16, counts
    assert len(empty) >= 3 and empty == list(range(empty[0], empty[-1] + 1))  # one contiguous empty stretch


@pytest.mark.parametrize("count", [512, 513])
def test_ground_row_contacts(reference, count):
    """Exactly `count` contacts from the first pass on: the next pass builds the hash from that table."""
    counts = [len(s["pairs"]) for s in _walk(reference, f"ground_row{count}")]
    assert counts == [count] * len(counts)


def test_brute_pairs_rules():
    """The pair rules of brute_pairs on hand-made boxes: closed overlap, same body, body types, filter, segments,
    joints."""
    f = np.float32
    fat = np.array([[0, 0, 1, 1], [1, 0, 2, 1], [np.nextafter(f(2), f(3)), 0, 3, 1], [0.5, 0.5, 1.5, 1.5],
                    [0, 0, 1, 1], [0, 0, 3, 1]], f)
    body = np.array([0, 1, 2, 3, 0, 4])
    btype = np.array([capi.DYNAMIC_BODY, capi.DYNAMIC_BODY, capi.DYNAMIC_BODY, capi.STATIC_BODY, capi.KINEMATIC_BODY])
    got = pe.brute_pairs(fat, body, btype)
    # 0-1 touch; 1-2 one ulp apart; 0-4 same body; 3 static with dynamic ok; 5 kinematic with dynamic ok
    assert got == {(0, 1), (0, 3), (1, 3), (3, 4), (0, 5), (1, 5), (2, 5), (4, 5), (1, 4)}
    filt = np.array([[1, 0xFFFFFFFF, 0]] * 6)
    filt[5] = [2, 0xFFFFFFFE, 0]  # category 2, does not collide with category 1
    assert (0, 5) not in pe.brute_pairs(fat, body, btype, filt)
    filt[[0, 1], 2] = -3  # same negative group: never
    assert (0, 1) not in pe.brute_pairs(fat, body, btype, filt)
    assert (0, 1) not in pe.brute_pairs(fat, body, btype, shape_type=np.array([3, 3, 2, 2, 2, 2]))
    assert (0, 1) not in pe.brute_pairs(fat, body, btype, joint_pairs=[(1, 0)])
