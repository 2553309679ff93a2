"""The CPU oracle against the UNMODIFIED reference's own roll-outs, bit for bit.

The reference was rolled out with seeded random actions — other seeds, batch sizes and scenario
arguments than the golden fixtures of ``tests/test_oracle_golden.py`` use — and at every step
``tests/make_golden.py`` recorded what the reference's ``World.step`` received and returned
(``tests/golden/reference/teacher_forced/``).  The oracle is teacher-forced on those inputs and must
return what the reference returned: bit for bit for the physics, the LIDAR readings and the distance /
overlap queries.  This is the pin the ``oracle/`` docstrings refer to.
"""
import itertools
import os

import pytest
import torch

import golden_pack
from golden_util import GOLDEN_DIR
from oracle import queries as Q
from oracle import world_step as WS
from vectorizedmultiagentsimulator_b200.simulator import plan as P

# name, kwargs, num_envs, steps, seed
CASES = [
    ("balance", dict(n_agents=3), 20, 30, 3),
    ("balance", dict(n_agents=5, package_mass=7), 9, 20, 4),
    ("transport", dict(n_agents=3, n_packages=2), 12, 20, 5),
    ("navigation", dict(n_agents=5), 12, 20, 6),
    ("flocking", dict(n_agents=4), 12, 15, 7),
    ("pollock", dict(lidar=True), 4, 6, 8),
    ("waterfall", dict(), 8, 12, 9),
    ("reverse_transport", dict(), 8, 12, 10),
    ("joint_passage", dict(), 6, 10, 11),
    ("wheel", dict(), 8, 12, 12),
    ("wind_flocking", dict(), 8, 10, 13),
    # crafted worlds (tests/crafted.py): action clamps, angular friction, joints with anchors apart,
    # a one-env batch without work items, 70 entities — branches no reference scenario takes
    ("crafted_clamps", dict(), 21, 15, 14),
    ("crafted_joints_apart", dict(), 10, 5, 15),
    ("crafted_lonely", dict(), 1, 5, 16),
    ("crafted_crowd", dict(), 3, 5, 17),
]
STATE = ("pos", "vel", "rot", "ang_vel")


def case_id(i, name):
    return f"{name}-{i}"


def _same(got, want, rec):
    """Bit for bit on the vector ISA the reference ran on (``rec``'s); elsewhere the last place of a
    transcendental may round differently (the 2e-6 of tests/test_oracle_golden.py)."""
    if rec["cpu_capability"] == torch.backends.cpu.get_cpu_capability() or got.dtype == torch.bool:
        return torch.equal(got, want)
    return got.shape == want.shape and (got.numel() == 0 or float((got - want).abs().max()) <= 2e-6)


@pytest.mark.parametrize("i", range(len(CASES)), ids=[case_id(i, c[0]) for i, c in enumerate(CASES)])
def test_oracle_equals_live_reference_bit_for_bit(i):
    name, _, _, steps, _ = CASES[i]
    rec = golden_pack.load(os.path.join(GOLDEN_DIR, "reference", "teacher_forced", case_id(i, name) + ".npz"))
    tables = P.build_tables(P.WorldDescription.from_json(rec["desc"]))
    assert len(rec["steps"]) == steps
    prev = None
    for t, entry in enumerate(rec["steps"]):
        state = {k: v.clone() for k, v in entry.get("state_in", prev).items() if k in STATE}
        state["force"], state["torque"] = entry["force"].clone(), entry["torque"].clone()
        want = entry["out"]
        gravity = entry["ent_gravity"]
        WS.world_step(tables, state, fixed_rot=entry["fixed_rot"], **({"ent_gravity": gravity} if gravity else {}))
        for k in STATE:
            assert _same(state[k], want[k], rec), f"{name} step {t}: {k} max |diff| {float((state[k] - want[k]).abs().max())}"
        prev = want
    for r in rec["lidar"]:
        want = rec["steps"][r["step"]]["out"]
        got = Q.cast_rays(tables, want["pos"], want["rot"], r["src"], r["targets"], r["angles"], r["max_range"])
        assert _same(got, r["out"], rec), f"{name} step {r['step']}: lidar of entity {r['src']}"
    # distance / overlap queries on the final state
    final = rec["final_state"]
    n_ents = final["pos"].shape[1]
    assert [(q["a"], q["b"]) for q in rec["queries"]] == list(itertools.permutations(range(n_ents), 2))[:40]
    for q in rec["queries"]:
        a, b = q["a"], q["b"]
        assert _same(Q.pair_distance(tables, final["pos"], final["rot"], a, b), q["distance"], rec)
        assert _same(Q.pair_overlap(tables, final["pos"], final["rot"], a, b), q["overlap"], rec)
        assert _same(Q.distance_from_point(tables, final["pos"], final["rot"], a, q["point"]), q["point_distance"], rec)
