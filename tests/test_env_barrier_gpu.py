"""The batch-wide broad phase of the one-kernel step (``step_env_kernel``) at its grid barrier.

Every block publishes its envs' masked bits and checks in at the barrier, but waits for the other blocks only if
its own envs left a masked bit unset; the last block to finish clears the mask region for the next launch.  The
captured one-launch step must still return, bit for bit, what the eager step and the two-launch step return.

The states are crafted so that the batch-wide bit matters: one line–sphere pair is placed, in every env, with the
sphere just beyond the circumscribed circles along the line's axis (the broad test says "far", yet the contact
reaches it), and the same pair is placed inside them in the envs that are to set the bit.  An env in the shell
gets a contact force exactly when some env of the batch sets the bit.  The cases run in the order every env →
no env → one env in the last block → one env in block 0, so a bit or an arrival left over from an earlier step
shows up as a wrong force; after each one the mask region must be all zero.  balance (1 substep) and transport
with 2 lines and 3 substeps (3 barriers per step), on lane pairs (G = 2) and, past what lane pairs hold at once,
one lane per env (G = 1).
"""
import pytest
import torch

import vectorizedmultiagentsimulator_b200 as b200
from envutil import flatten, sync_env
from golden_util import same_result
from vectorizedmultiagentsimulator_b200 import _native
from vectorizedmultiagentsimulator_b200.simulator import plan as P
from vectorizedmultiagentsimulator_b200.simulator.core import Line, Sphere
from vectorizedmultiagentsimulator_b200.simulator.environment import environment as E

pytestmark = pytest.mark.gpu

EXACT = _native.ARITH == "exact"
SLAB = ("pos", "vel", "rot", "ang_vel", "force", "torque")
BLOCK = 64  # envs per block of step_env_kernel, whatever the lanes per env
SHELL = 1e-4  # beyond the circumscribed circles, inside the contact margin

CONFIGS = {
    "balance": ("balance", dict(n_agents=4)),
    "transport3": ("transport", dict(n_agents=4, n_lines=2, substeps=3)),
}


def _make(name, n, monkeypatch, flags=None, cuda_graph=True):
    scenario, kwargs = CONFIGS[name]
    with monkeypatch.context() as m:
        for k, v in (flags or {}).items():
            m.setattr(E, k, v)
        m.setattr(E, "_WHOLE_STEP_KERNEL_WAIT_S", 600.0)
        env = b200.make_env(scenario, num_envs=n, device="cuda", seed=0, cuda_graph=cuda_graph, **kwargs)
        env.reset()
        if cuda_graph:  # (warm-up steps and the capture happen here, while the flags are set)
            gen = torch.Generator().manual_seed(1)
            for _ in range(4):
                env.step(_actions(env, gen))
    return env


def _actions(env, gen):
    return [((torch.rand(env.num_envs, a.action_size, generator=gen) * 2 - 1) * a.action.u_range_tensor.cpu()).cuda()
            for a in env.agents]


def _same(g, w):
    if not EXACT:
        return same_result(g.float(), w.float(), atol=2e-4)
    if g.shape != w.shape or g.dtype != w.dtype:
        return False
    if not g.is_floating_point():
        return torch.equal(g, w)
    return bool(((g == w) | (g.isnan() & w.isnan())).all())


def _line_sphere_item(env):
    """(item, line entity, sphere entity, broad threshold) of the first masked line–sphere pair with a movable sphere."""
    tables = env.world._get_backend().tables
    ents = env.world.entities
    for k in range(tables.n_masked):
        item = int(tables.masked_items[k])
        a, b = (int(v) for v in tables.item_i32[item, 1:3])
        for line, sphere in ((a, b), (b, a)):
            if isinstance(ents[line].shape, Line) and isinstance(ents[sphere].shape, Sphere) and ents[sphere].movable:
                return item, line, sphere, float(tables.item_f32[item, P.IF_BROAD_THR])
    raise AssertionError("no masked line–sphere pair")


def _craft(env, near):
    """Puts the pair's sphere on the line's axis, just beyond the circumscribed circles in every env and inside
    them in the envs of ``near`` (a bool [B] mask)."""
    item, line, sphere, thr = _line_sphere_item(env)
    slab = env.world.slab
    with torch.no_grad():
        slab.rot[:, line] = 0.0
        slab.ang_vel[:, line] = 0.0
        off = torch.full((env.num_envs,), thr + SHELL, device=slab.pos.device)
        off[near.to(off.device)] = thr - SHELL
        slab.pos[:, sphere, 0] = slab.pos[:, line, 0] + off
        slab.pos[:, sphere, 1] = slab.pos[:, line, 1]
        slab.vel[:, sphere] = 0.0
    # the broad test in float64 terms of the kernel's: which envs set the bit
    d = torch.linalg.vector_norm(slab.pos[:, line] - slab.pos[:, sphere], dim=-1)
    assert torch.equal(d <= thr, near.to(d.device)), "the crafted pair does not set the bit where intended"


def _mask_region(env):
    return env.world._get_backend()._dev_tables.mask


def _cases(n):
    near_all = torch.ones(n, dtype=torch.bool)
    near_none = torch.zeros(n, dtype=torch.bool)
    last = torch.zeros(n, dtype=torch.bool)
    last[n - 1] = True  # (the last block: n is not a multiple of the block, so it is a partial one)
    first = torch.zeros(n, dtype=torch.bool)
    first[BLOCK // 2] = True
    return [("every env", near_all), ("no env", near_none), ("one env, last block", last), ("one env, block 0", first)]


def _run(name, n, monkeypatch, two_launches=True, steps=3):
    envs = {"eager": _make(name, n, monkeypatch, cuda_graph=False), "one kernel": _make(name, n, monkeypatch)}
    if two_launches:
        envs["two launches"] = _make(name, n, monkeypatch, dict(_INGEST_IN_KERNEL=False))
    ref, one = envs["eager"], envs["one kernel"]
    plan = one._one_call
    assert plan is not None and plan.c.ingest_in_kernel == 1 and plan.c.fused_kernel > 0, "not one launch"
    if two_launches:
        assert envs["two launches"]._one_call.c.ingest_in_kernel == 0
    assert n % BLOCK != 0
    gen = torch.Generator().manual_seed(5)
    backend = one.world._get_backend()
    for label, near in _cases(n):
        _craft(ref, near)
        for env in envs.values():
            if env is not ref:
                sync_env(ref, env)
        for t in range(steps):
            actions = _actions(ref, gen)
            want = ref.step([a.clone() for a in actions])
            for what, env in envs.items():
                if env is ref:
                    continue
                before = backend.launches
                got = env.step([a.clone() for a in actions])
                if env is one:
                    assert backend.launches - before == 1, f"{label} step {t}: {backend.launches - before} launches"
                tag = f"{name} {n} envs, {label}, {what} step {t}"
                for i, (g, w) in enumerate(zip(flatten(got), flatten(want))):
                    assert g.dtype == w.dtype and _same(g, w), f"{tag}: output leaf {i}"
                for k in SLAB:
                    assert _same(getattr(env.world.slab, k), getattr(ref.world.slab, k)), f"{tag}: slab {k}"
                for a, b in zip(env.agents, ref.agents):
                    assert _same(a.action.u, b.action.u), f"{tag}: {a.name} action.u"
                env.check_actions_now()  # (the bad-action flag stays clear, as on the eager step)
                if not EXACT:
                    sync_env(ref, env)
            torch.cuda.synchronize()
            region = _mask_region(one)
            assert int(region.abs().sum()) == 0, f"{name} {label} step {t}: mask region not cleared: {region.tolist()}"


@pytest.mark.parametrize("name", list(CONFIGS))
def test_barrier_lane_pairs(name, monkeypatch):
    # 8 blocks and a partial one: G = 2
    _run(name, 8 * BLOCK + 17, monkeypatch)


@pytest.mark.parametrize("name", list(CONFIGS))
def test_barrier_one_lane_per_env(name, monkeypatch):
    """Past what lane pairs hold at once (4 blocks of 128 threads per SM), one lane per env, still one launch."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    _run(name, sms * 4 * BLOCK + BLOCK + 17, monkeypatch, two_launches=False, steps=2)
