"""CPU companion of tests/test_hub_capacity_gpu.py: every hub scene (tests/hub_cases.py), built and collided by the
reference, reaches exactly the sizes the GPU cases rely on: the serial group's contacts, joints and distinct bodies, each
hub's incidence-list length and the number of hubs. A scene that drifts off its edge fails here, without a GPU."""
import numpy as np
import pytest

import hub_cases
from hub_cases import SCENES, build_rows, check_sizes, degrees, serial_sizes


@pytest.mark.parametrize("name", sorted(SCENES))
def test_scene_reaches_its_sizes(reference, name):
    bodies, contacts, joints, sc = build_rows(reference, name, "TGS_Soft")
    check_sizes(name, bodies, contacts, joints)
    live = contacts["pointCount"] > 0
    assert live.all(), "every contact the scenes make has points"


@pytest.mark.parametrize("name", ["contacts_2049", "joints_257", "lists"])
def test_hubs_are_body_a_and_body_b(reference, name):
    """The hub is body A of some of its constraints and body B of others, so both sides of the incidence entry are sorted."""
    bodies, contacts, joints, sc = build_rows(reference, name, "TGS_Soft")
    deg = degrees(bodies, contacts, joints)
    for hub in np.nonzero(deg > hub_cases.HEAVY_DEGREE)[0]:
        jl = (joints["flags"] & 1) == 1
        as_a = int((contacts["bodyA"] == hub).sum() + (joints["bodyA"][jl] == hub).sum())
        as_b = int((contacts["bodyB"] == hub).sum() + (joints["bodyB"][jl] == hub).sum())
        assert as_a > 0 and as_b > 0 and as_a + as_b == deg[hub], (name, hub, as_a, as_b)


def test_serial_sizes_follow_the_threshold(reference):
    """The thresholds the disagreement cases run under: the serial group at S2B_HUB_DEGREE 100, 30 and the default."""
    b, c, j, _ = build_rows(reference, "degree_60", "TGS_Soft")
    assert serial_sizes(b, c, j, hub_degree=100) == (0, 0, 0)
    assert serial_sizes(b, c, j) == (60, 0, 2)
    b, c, j, _ = build_rows(reference, "degree_40", "TGS_Soft")
    assert serial_sizes(b, c, j, hub_degree=30) == (40, 0, 2)
    assert serial_sizes(b, c, j) == (0, 0, 0)
    b, c, j, _ = build_rows(reference, "degree_48_49", "TGS_Soft")
    assert serial_sizes(b, c, j) == (49, 0, 2)
    b, c, j, _ = build_rows(reference, "colour_limit", "TGS_Soft")
    assert serial_sizes(b, c, j, hub_degree=0) == (0, 0, 0)
    assert degrees(b, c, j).max() == 100


@pytest.mark.parametrize("solver", ["Jacobi", "PGS", "PGS_NGS", "PGS_NGS_Block", "PGS_Soft", "SoftStep", "TGS_Sticky", "TGS_NGS",
                                    "XPBD"])
def test_sizes_do_not_depend_on_the_variant(reference, solver):
    """The GPU cases build each scene for the variant they run."""
    for name in sorted(SCENES):
        b, c, j, _ = build_rows(reference, name, solver)
        check_sizes(name, b, c, j)
