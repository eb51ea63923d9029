"""GPU: the pair search at its capacity edges (tests/pair_edges.py), every step against the reference and against a
brute-force restatement of the pair table.

Every case runs through test_multistep_gpu._run (the reference's collide, the oracle replayed in the device's order, the
reference's finalize; pair set and (A, B) order, manifolds, bodies, shape and fat boxes compared with tolerance 0),
under S2B_FINALIZE_REFIT 0 / 1 times S2B_PREFETCH_PAIRS 0 / 1. Every step the device's table also equals
pair_edges.brute_pairs over the device's own fat boxes as that step's pass saw them, on every pass that built the
hierarchy treeHeight equals pair_edges.restated_height over the same boxes, and the four runs' contact tables and bodies
are byte-identical: the pairs a proxy finds do not depend on the route it takes. Each case asserts through s2bCounters
(pairRetries, prefetchRetries, largeMovers, treeBuilds, finalizeRefits) which side of its edge it reached."""
import contextlib
import os

import pytest

import pair_edges as pe
from solver2d_b200 import capi, device
from test_multistep_gpu import _run

pytestmark = pytest.mark.gpu
CONFIGS = [(refit, prefetch) for refit in (0, 1) for prefetch in (0, 1)]


@pytest.fixture(scope="module")
def product():
    return capi.Solver2D(device.LIB_PATH)


@contextlib.contextmanager
def _env(**values):
    old = {k: os.environ.get(k) for k in values}
    os.environ.update({k: str(v) for k, v in values.items()})
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v


def _case(reference, product, dev, name, buffer=None, solver="TGS_Soft", configs=CONFIGS):
    """Run scene `name` under `configs`; per configuration the counters after every step. Checks every step the
    brute-force pair set and, on a step whose pass built the hierarchy, treeHeight against the restated height over
    the fat boxes that pass saw; then the byte identity of the runs."""
    builder, steps = pe.SCENES[name]
    runs = {}
    for refit, prefetch in configs:
        held = {}

        def recipe(lib, solver):
            sc = builder(lib, solver)
            if lib is product:
                held["sc"] = sc
            return sc

        seen, tables = [], []
        hook = pe.before_step_for(name)

        def setup(dw):
            held["dw"] = dw
            held["fat"] = pe.device_fat(dw)

        def before_step(step, worlds):
            # the pass of a step sees the fat boxes as the step before left them, or as uploaded since
            if hook is not None:
                hook(step, worlds)
                product.s2World_Flush(worlds[1][1].world)
                held["fat"] = pe.device_fat(held["dw"])

        def after_step(dw):
            step = len(seen)
            fat, live = held["fat"]
            want, got = pe.device_pairs(product, held["sc"], dw, fat)
            held["fat"] = pe.device_fat(dw)
            assert want == got, f"{name} refit={refit} prefetch={prefetch} step {step}: brute force != device: " \
                                f"missing {sorted(want - got)[:5]}, extra {sorted(got - want)[:5]}"
            c = dw.counters()
            if c.treeBuilds > (seen[-1].treeBuilds if seen else 0):
                assert c.treeHeight == pe.restated_height(fat, live), (name, refit, prefetch, step, c.treeHeight)
            seen.append(c)
            tables.append((dw.download_contacts(c.contactCount).tobytes(), dw.download_all_bodies(c.bodyCapacity).tobytes()))

        knobs = dict(S2B_FINALIZE_REFIT=refit, S2B_PREFETCH_PAIRS=prefetch)
        if buffer is not None:
            knobs["S2B_PAIR_BUFFER"] = buffer
        with _env(**knobs):
            _run(reference, product, dev, recipe, solver, steps, 4, 2, {}, setup=setup, before_step=before_step,
                 after_step=after_step)
        runs[(refit, prefetch)] = (seen, tables)
    base = runs[configs[0]][1]
    for cfg in configs[1:]:
        for step, (a, b) in enumerate(zip(base, runs[cfg][1])):
            assert a[0] == b[0], f"{name} {cfg} step {step}: contact table differs from refit=0 prefetch=0"
            assert a[1] == b[1], f"{name} {cfg} step {step}: bodies differ from refit=0 prefetch=0"
    return {cfg: r[0] for cfg, r in runs.items()}


def test_lattice_burst_reruns_the_synchronous_search(reference, product, dev):
    """1 500 boxes created in one go into a world whose pair buffer was sized for 4 shape slots: the step's search (never
    a prefetched one: the shapes were uploaded) overflows and runs once more. The shape pool grew, so the hierarchy is
    rebuilt and no refit finalize made is taken over."""
    k = pe.LATTICE_STEP
    for cfg, seen in _case(reference, product, dev, "lattice_burst").items():
        before, after = seen[k - 1], seen[k]
        assert after.pairRetries == before.pairRetries + 1, cfg
        assert seen[-1].pairRetries == 1 and seen[-1].prefetchRetries == 0, cfg
        assert after.shapeCapacity > before.shapeCapacity
        assert after.treeBuilds > before.treeBuilds, cfg
        assert after.finalizeRefits == before.finalizeRefits, cfg
        if cfg[0] == 1:
            assert before.finalizeRefits > 0, cfg  # the passes before took finalize's refit


def test_interleaving_clouds_rerun_the_prefetched_search(reference, product, dev):
    """S2B_PAIR_BUFFER = 64: the first burst of new pairs overflows the search started behind the step before (prefetch
    on) or the step's own search (prefetch off); both are run again, with the same results."""
    for (refit, prefetch), seen in _case(reference, product, dev, "interleaving_clouds", buffer=pe.CLOUD_BUFFER).items():
        last = seen[-1]
        if prefetch:
            assert last.prefetchRetries >= 1 and last.pairRetries == last.prefetchRetries, (refit, prefetch)
        else:
            assert last.prefetchRetries == 0 and last.pairRetries == 1, (refit, prefetch)


@pytest.mark.parametrize("name,large", [("large_glide64", 64), ("large_glide65", 65)])
def test_large_movers_every_pass(reference, product, dev, name, large):
    """64 / 65 large movers on every pass, fused or not (the 65th walks the hierarchy); every one of them overlaps
    static boxes, which never query, so a lost large mover loses pairs."""
    for cfg, seen in _case(reference, product, dev, name).items():
        assert [c.largeMovers for c in seen] == [large] * len(seen), cfg
        if cfg[0] == 1:
            assert seen[-1].finalizeRefits > 0, cfg


@pytest.mark.parametrize("name,large", [("one_big255", 0), ("one_big256", 1)])
def test_large_mover_leaf_threshold(reference, product, dev, name, large):
    """255 / 256 leaves: no large-mover route below 256, counted on the first pass, where every movable shape moved."""
    for cfg, seen in _case(reference, product, dev, name).items():
        assert seen[0].largeMovers == large, (cfg, seen[0].largeMovers)


def test_root_box_changing_between_passes(reference, product, dev):
    """The marker raises the root box every step. On ROOT_FLIP_STEP the fused path (previous refit's root) routes the
    slider as a large mover and the unfused search (the pass's own root) walks it; same pairs either way."""
    k = pe.ROOT_FLIP_STEP
    for cfg, seen in _case(reference, product, dev, "root_flip").items():
        fused = seen[k].finalizeRefits > seen[k - 1].finalizeRefits
        assert fused == (cfg[0] == 1), cfg
        assert seen[k].largeMovers == (1 if fused else 0), (cfg, seen[k].largeMovers)
        assert seen[k - 1].largeMovers == 1 and seen[k + 1].largeMovers == 0, cfg


@pytest.mark.parametrize("name", ["line_row", "far_pile", "cluster"])
def test_degenerate_morton_inputs(reference, product, dev, name):
    """Centres on one line (zero-height axis clamped to 1e-6), a pile 1e4 m from the origin, a staircase cluster with
    duplicate codes: treeHeight equals the restated height (checked in _case on every building pass), pairs exact."""
    for cfg, seen in _case(reference, product, dev, name).items():
        assert seen[0].treeBuilds >= 1 and seen[0].treeHeight > 0, cfg


def test_rebuild_cadence(reference, product, dev):
    """The slider stops and starts every 3 steps: passes on half of the steps, finalize refits left unused on the still
    steps, periodic rebuilds; every rebuild's height restated, pairs exact."""
    for cfg, seen in _case(reference, product, dev, "cadence").items():
        last = seen[-1]
        assert last.pairPassCount > 17 and last.treeBuilds >= 2, (cfg, last.pairPassCount, last.treeBuilds)
        passes = [c.pairPassCount for c in seen]
        assert any(b == a for a, b in zip(passes, passes[1:])), cfg  # still steps without a pass
        if cfg[0] == 1:
            assert 0 < last.finalizeRefits < last.pairPassCount, cfg


OTHER_VARIANTS = [s for s in capi.SOLVER_TYPES if s != "TGS_Soft"]


@pytest.mark.parametrize("solver", OTHER_VARIANTS)
def test_large_movers_and_prefetched_rerun_other_variants(reference, product, dev, solver):
    """The pair search does not depend on the solver variant, but the finalize before it does: the 65-mover glide and the
    prefetched re-run under every other variant, fused refit and prefetch on."""
    seen = _case(reference, product, dev, "large_glide65", solver=solver, configs=[(1, 1)])[(1, 1)]
    assert [c.largeMovers for c in seen] == [65] * len(seen) and seen[-1].finalizeRefits > 0
    seen = _case(reference, product, dev, "interleaving_clouds", buffer=pe.CLOUD_BUFFER, solver=solver, configs=[(1, 1)])[(1, 1)]
    assert seen[-1].prefetchRetries >= 1


def test_exact_touch(reference, product, dev):
    """Fat boxes touching exactly pair, and survive every pass while touching; the neighbour one ulp off never pairs."""
    for cfg, seen in _case(reference, product, dev, "exact_touch").items():
        assert seen[-1].pairPassCount >= len(seen) and seen[-1].contactCount == 4, cfg


def test_launched_row_empties_and_refills(reference, product, dev):
    """Boxes thrown up off the ground: the table empties, passes run on an empty table, and the contacts come back."""
    for cfg, seen in _case(reference, product, dev, "launched_row").items():
        counts = [c.contactCount for c in seen]
        empty = [k for k, n in enumerate(counts) if n == 0]
        assert empty and counts[-1] == 16, (cfg, counts)
        passes = [c.pairPassCount for c in seen]
        # a pass ran over the empty table: a step after an empty step that ran a pass
        assert any(k - 1 in empty and passes[k] > passes[k - 1] for k in empty), cfg


@pytest.mark.parametrize("count", [512, 513])
def test_ground_row_hash_sizes(reference, product, dev, count):
    """`count` contacts from the first pass on; the second pass builds the pair-key hash from that table (1 024 slots for
    512 contacts, 2 048 for 513)."""
    for cfg, seen in _case(reference, product, dev, f"ground_row{count}").items():
        assert [c.contactCount for c in seen] == [count] * len(seen), cfg
        assert seen[1].pairPassCount > seen[0].pairPassCount, cfg
