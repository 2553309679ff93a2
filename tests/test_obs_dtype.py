"""16-bit observations (``make_env(..., obs_dtype=torch.float16 | torch.bfloat16)``) on the CPU oracle backend.

Every fp32 leaf of every observation an environment hands out must be exactly ``leaf.to(obs_dtype)`` of what the
same environment with fp32 observations hands out, and nothing else may change: rewards, dones, infos and the
state slab stay bit-identical.  Each case steps an fp32 env and a 16-bit env built with the same seed through the
same actions, a masked (or indexed) reset and, where the scenario supports it, ``auto_reset``.  The kernels that do
the rounding on the GPU are checked in tests/test_obs_dtype_gpu.py and tests/test_obs_dtype_hostsim.py.
"""
import numpy as np
import pytest
import torch

import stock_style
import vectorizedmultiagentsimulator_b200 as b200
from envutil import flatten
from oracle.backend import use_oracle

N_ENVS = 24
STEPS = 20
DTYPES = [torch.float16, torch.bfloat16]
BITS = {torch.float16: torch.int16, torch.bfloat16: torch.int16, torch.float32: torch.int32}

CASES = [
    ("balance", dict(n_agents=4)),
    ("transport", dict(n_agents=4)),
    ("navigation", dict(n_agents=3)),
    ("flocking", dict(n_agents=4)),
    ("stock_style", dict(n_agents=3)),
]


def _scenario(name):
    return stock_style.make_scenario() if name == "stock_style" else name


def assert_rounded(got, want32, dtype, what):
    """``got`` is ``want32.to(dtype)`` bit for bit, NaN where ``want32`` is NaN (any payload)."""
    assert got.dtype == dtype and got.shape == want32.shape, what
    want = want32.to(dtype)
    nan = want32.isnan()
    assert torch.equal(got.isnan(), nan), f"{what}: NaN positions"
    assert torch.equal(got.view(BITS[dtype])[~nan], want.view(BITS[dtype])[~nan]), f"{what}: bits"


def assert_same(got, want, what):
    assert got.dtype == want.dtype and got.shape == want.shape, what
    if got.is_floating_point():
        nan = want.isnan()
        assert torch.equal(got.isnan(), nan), f"{what}: NaN positions"
        assert torch.equal(got.view(BITS[got.dtype])[~nan], want.view(BITS[want.dtype])[~nan]), f"{what}: bits"
    else:
        assert torch.equal(got, want), what


def assert_obs(got, want, dtype, what):
    """One observation structure (list / dict of per-agent tensors or dicts)."""
    g, w = flatten(got), flatten(want)
    assert len(g) == len(w), what
    for i, (x, y) in enumerate(zip(g, w)):
        if y.dtype == torch.float32:
            assert_rounded(x, y, dtype, f"{what} leaf {i}")
        else:
            assert_same(x, y, f"{what} leaf {i}")


def _roll(name, kwargs, obs_dtype, auto_reset, **env_kw):
    """Everything the env hands out over a seeded roll-out, and the slab after every call."""
    with use_oracle():
        env = b200.make_env(_scenario(name), num_envs=N_ENVS, device="cpu", seed=3, obs_dtype=obs_dtype,
                            auto_reset=auto_reset, max_steps=6 if auto_reset else None, **env_kw, **kwargs)
        masked = env.scenario.supports_masked_reset
        out = [("reset", env.reset(seed=3))]
        gen = torch.Generator().manual_seed(7)
        slabs = []
        for t in range(STEPS):
            actions = [(torch.rand(N_ENVS, env.get_agent_action_size(a), generator=gen) * 2 - 1) for a in env.agents]
            out.append((f"step {t}", env.step(actions)))
            if t == 9:
                mask = torch.zeros(N_ENVS, dtype=torch.bool)
                mask[::5] = True
                out.append(("reset_at", env.reset_at(mask if masked else 4)))
            slabs.append({k: v.clone() for k, v in env.world.slab.state_dict().items()})
    return env, out, slabs


def _check_pair(name, kwargs, dtype, auto_reset, **env_kw):
    env32, want, slabs32 = _roll(name, kwargs, torch.float32, auto_reset, **env_kw)
    env16, got, slabs16 = _roll(name, kwargs, dtype, auto_reset, **env_kw)
    assert env16.obs_dtype == dtype
    for (label, g), (_, w) in zip(got, want):
        if label in ("reset", "reset_at"):
            assert_obs(g, w, dtype, f"{name} {label} obs")
            continue
        assert_obs(g[0], w[0], dtype, f"{name} {label} obs")
        for k, (x, y) in enumerate(zip(flatten(g[1:]), flatten(w[1:]))):
            assert_same(x, y, f"{name} {label} result {k}")
    for t, (a, b) in enumerate(zip(slabs16, slabs32)):
        for k in a:
            assert_same(a[k], b[k], f"{name} step {t} slab {k}")
    return env16, got


@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("name,kwargs", CASES, ids=[c[0] for c in CASES])
def test_observations_are_the_fp32_observations_rounded(name, kwargs, dtype):
    env, got = _check_pair(name, kwargs, dtype, auto_reset=False)
    obs = got[1][1][0]
    assert all(o.dtype == dtype for o in obs)
    assert all(r.dtype == torch.float32 for r in got[1][1][1])
    if env.scenario.supports_masked_reset:
        # auto_reset: a finished env hands out the (rounded) first observation of its next episode
        _check_pair(name, kwargs, dtype, auto_reset=True)


@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
def test_dict_spaces(dtype):
    env, got = _check_pair("balance", dict(n_agents=3), dtype, auto_reset=False, dict_spaces=True)
    obs = got[1][1][0]
    assert isinstance(obs, dict) and set(obs) == {a.name for a in env.agents}
    assert all(v.dtype == dtype for v in obs.values())


def _dict_obs_scenario():
    """stock_style with dict observations: an fp32 leaf, a nested fp32 leaf, a bool and an int64 leaf."""
    sc = stock_style.make_scenario()
    flat = sc.observation

    def observation(agent):
        x = flat(agent)
        return {"x": x, "nested": {"pos": agent.state.pos}, "near": x[:, 0] > 0, "count": (x[:, :2] > 0).sum(-1)}

    sc.observation = observation
    return sc


@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
def test_dict_observations_round_only_their_fp32_leaves(dtype):
    outs = {}
    for d in (torch.float32, dtype):
        with use_oracle():
            env = b200.make_env(_dict_obs_scenario(), num_envs=N_ENVS, device="cpu", seed=1, obs_dtype=d, n_agents=2)
            gen = torch.Generator().manual_seed(2)
            outs[d] = [env.reset(seed=1)]
            for _ in range(3):
                outs[d].append(env.step([torch.rand(N_ENVS, 2, generator=gen) * 2 - 1 for _ in env.agents])[0])
            outs[d].append(env.reset_at(1))
    for t, (g, w) in enumerate(zip(outs[dtype], outs[torch.float32])):
        assert_obs(g, w, dtype, f"call {t}")
        o = g[0]
        assert o["x"].dtype == dtype and o["nested"]["pos"].dtype == dtype
        assert o["near"].dtype == torch.bool and o["count"].dtype == torch.int64
    space = env.observation_space[0]
    assert set(space.spaces) == {"x", "nested", "near", "count"}


def test_observation_spaces():
    want = {torch.float32: np.float32, torch.float16: np.float16, torch.bfloat16: np.float32}
    for dtype, np_dtype in want.items():
        with use_oracle():
            env = b200.make_env("balance", num_envs=4, device="cpu", seed=0, obs_dtype=dtype, n_agents=3)
        for space, obs in zip(env.observation_space, env.reset()):
            assert space.dtype == np_dtype and space.shape == obs.shape[1:]
            assert np.isinf(space.low).all() and np.isinf(space.high).all()


def test_bad_obs_dtypes_are_refused():
    with use_oracle():
        for bad in (torch.float64, torch.int32, "float16", np.float16):
            with pytest.raises(ValueError, match="torch.float32, torch.float16 or torch.bfloat16"):
                b200.make_env("balance", num_envs=4, device="cpu", seed=0, obs_dtype=bad, n_agents=3)
        with pytest.raises(ValueError, match="bfloat16"):
            b200.make_env("balance", num_envs=4, device="cpu", seed=0, obs_dtype=torch.bfloat16, wrapper="gym",
                          n_agents=3)


def test_float16_through_a_wrapper():
    with use_oracle():
        bare = b200.make_env("balance", num_envs=1, device="cpu", seed=0, n_agents=3)
        env = b200.make_env("balance", num_envs=1, device="cpu", seed=0, n_agents=3, wrapper="gym",
                            obs_dtype=torch.float16)
        obs = env.reset(seed=4)
        bare.seed(4)
        want = bare.reset_at(index=0)
    assert obs[0].dtype == np.float16
    assert np.array_equal(obs[0].view(np.int16), want[0][0].to(torch.float16).numpy().view(np.int16))


def test_obs_dtype_is_an_explicit_argument_everywhere():
    import inspect

    from vectorizedmultiagentsimulator_b200 import shard
    from vectorizedmultiagentsimulator_b200.simulator.environment import Environment

    for fn in (b200.make_env, Environment.__init__, shard.make_shard_env):
        p = inspect.signature(fn).parameters["obs_dtype"]
        assert p.default is torch.float32 and p.kind is inspect.Parameter.POSITIONAL_OR_KEYWORD
