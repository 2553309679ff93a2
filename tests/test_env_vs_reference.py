"""The host layer (Environment / World object model / re-written scenarios) against the
UNMODIFIED reference's roll-outs, both on CPU: this package runs on the CPU oracle backend, so any
difference comes from the host code (action decoding, reset draws, obs/reward layout).  What the
reference returned is stored in ``tests/golden/reference/env/`` (``tests/make_golden.py``)."""
import functools
import os

import pytest
import torch

import golden_pack
from golden_util import GOLDEN_DIR
from oracle.backend import use_oracle

CASES = [
    ("balance", dict(n_agents=4)),
    ("transport", dict(n_agents=4)),
    ("navigation", dict(n_agents=8)),
    ("flocking", dict(n_agents=5)),
]

@functools.lru_cache(maxsize=None)
def _reference(case):
    return golden_pack.load(os.path.join(GOLDEN_DIR, "reference", "env", case + ".npz"))


def _flatten(x):
    if isinstance(x, dict):
        return [v for k in sorted(x) for v in _flatten(x[k])]
    if isinstance(x, (list, tuple)):
        return [v for item in x for v in _flatten(item)]
    return [x]


def _assert_same(got, want, what, tol=0.0, ref=None):
    """``want``: the reference's flattened leaves, from the fixture ``ref``.  ``tol`` holds on the vector ISA
    the reference ran on; elsewhere the last place of a transcendental may round differently (the 2e-6 of
    tests/test_oracle_golden.py)."""
    if ref["cpu_capability"] != torch.backends.cpu.get_cpu_capability():
        tol = max(tol, 2e-6)
    g, w = _flatten(got), want
    assert len(g) == len(w), what
    for a, b in zip(g, w):
        assert a.shape == b.shape and a.dtype == b.dtype, f"{what}: {a.shape}/{a.dtype} vs {b.shape}/{b.dtype}"
        if a.dtype == torch.bool:
            assert torch.equal(a, b), what
        else:
            assert float((a - b).abs().max()) <= tol, f"{what}: {float((a - b).abs().max())}"


@pytest.mark.parametrize("name,kwargs", CASES)
@pytest.mark.parametrize("continuous", [True, False])
def test_rollout_matches_reference(name, kwargs, continuous):
    import vectorizedmultiagentsimulator_b200 as b200

    ref = _reference(f"{name}-{'continuous' if continuous else 'discrete'}")
    n_envs, steps = 12, 12
    assert len(ref["steps"]) == steps
    with use_oracle():
        mine = b200.make_env(name, num_envs=n_envs, device="cpu", seed=3, continuous_actions=continuous, **kwargs)
        _assert_same(mine.reset(seed=5), ref["reset"], f"{name} reset obs", ref=ref)
        gen = torch.Generator().manual_seed(11)
        for t in range(steps):
            if continuous:
                actions = [
                    (torch.rand(n_envs, a.action_size, generator=gen) * 2 - 1) * a.action.u_range_tensor
                    for a in mine.agents
                ]
            else:
                actions = [torch.randint(0, 9, (n_envs, 1), generator=gen) for _ in mine.agents]
            got = mine.step([a.clone() for a in actions])
            for part, label in zip(range(4), ("obs", "rews", "dones", "infos")):
                _assert_same(got[part], ref["steps"][t][part], f"{name} step {t} {label}", tol=1e-6, ref=ref)
            if t == 5:  # partial reset mid-rollout (ref tests/test_vmas.py:249-262)
                _assert_same(mine.reset_at(2), ref["reset_at"], f"{name} reset_at obs", tol=1e-6, ref=ref)


def test_stock_style_scenario_matches_reference():
    """tests/stock_style.py — per-agent is_overlapping / get_distance / Lidar.measure callbacks as the
    reference's scenario files write them — built from this package's modules against the roll-out of the
    same scenario built from the reference's: identical roll-outs (this is the CPU half of the pin;
    tests/test_env_gpu.py steps the same scenario on the CUDA backend against the oracle env)."""
    import stock_style
    import vectorizedmultiagentsimulator_b200 as b200

    ref = _reference("stock_style")
    n_envs = 10
    with use_oracle():
        mine = b200.make_env(stock_style.make_scenario(), num_envs=n_envs, device="cpu", seed=1, n_agents=3)
        gen = torch.Generator().manual_seed(2)
        for t in range(10):
            actions = [(torch.rand(n_envs, a.action_size, generator=gen) * 2 - 1) for a in mine.agents]
            got = mine.step([a.clone() for a in actions])
            for part, label in zip(range(4), ("obs", "rews", "dones", "infos")):
                _assert_same(got[part], ref["steps"][t][part], f"stock_style step {t} {label}", tol=0.0, ref=ref)
            if t == 4:
                _assert_same(mine.reset_at(3), ref["reset_at"], "stock_style reset_at obs", tol=0.0, ref=ref)


def test_dynamics_zoo_matches_reference():
    """tests/crafted.py "dynamics_zoo": one agent per action model (differential drive RK4 / Euler,
    kinematic bicycle, drone, forward, rotation, holonomic with rotation, static) — the host-side torch
    formulation of this package against the reference's, bit for bit.  (The CUDA ingest kernel that fuses
    them is checked against this formulation in tests/test_env_gpu.py.)"""
    import crafted
    import vectorizedmultiagentsimulator_b200 as b200

    ref = _reference("dynamics_zoo")
    n_envs = 9
    with use_oracle():
        mine = b200.make_env(
            crafted.make_scenario("vectorizedmultiagentsimulator_b200", "dynamics_zoo"), num_envs=n_envs, device="cpu", seed=2
        )
        gen = torch.Generator().manual_seed(3)
        for t in range(8):
            actions = [(torch.rand(n_envs, a.action_size, generator=gen) * 2 - 1) * a.action.u_range_tensor for a in mine.agents]
            got = mine.step([a.clone() for a in actions])
            want = ref["steps"][t]
            _assert_same(got[0], want["obs"], f"dynamics_zoo step {t} obs", tol=0.0, ref=ref)
            assert len(want["force"]) == len(mine.agents)
            for a_mine, force, torque in zip(mine.agents, want["force"], want["torque"]):
                _assert_same(a_mine.state.force, [force], f"step {t}: force of {a_mine.name}", ref=ref)
                _assert_same(a_mine.state.torque, [torque], f"step {t}: torque of {a_mine.name}", ref=ref)


def test_spaces_and_random_actions_match_reference():
    import vectorizedmultiagentsimulator_b200 as b200

    ref = _reference("spaces")
    with use_oracle():
        mine = b200.make_env("balance", num_envs=4, device="cpu", seed=0, n_agents=3)
    assert len(mine.action_space.spaces) == ref["n_action_spaces"] == 3
    assert tuple(mine.observation_space.spaces[0].shape) == ref["observation_shape"]
    mine.seed(1)
    _assert_same(mine.get_random_actions(), ref["random_actions"], "random actions", ref=ref)


def test_seed_isolation_from_global_rng():
    """Env draws must not disturb the user's global torch RNG (ref tests/test_vmas.py:308-323)."""
    import vectorizedmultiagentsimulator_b200 as b200

    torch.manual_seed(123)
    expected = torch.rand(3)
    torch.manual_seed(123)
    with use_oracle():
        env = b200.make_env("navigation", num_envs=4, device="cpu", seed=0, n_agents=3)
        env.step(env.get_random_actions())
    assert torch.equal(torch.rand(3), expected)
