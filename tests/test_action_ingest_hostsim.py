"""The action ingest's device code (``ingest_actions_body<KIN>`` in csrc/ingest.cuh) run on the CPU, at its edges,
against the float64 reference of tests/action_ref.py and against the torch host path of the CPU oracle env
(``Environment._set_action`` and the dynamics' ``process_action``).

* Continuous actions: +-0, +-r, the neighbours of +-r, +-inf, NaN, +-FLT_MAX and the smallest subnormal, for several
  ranges and multipliers, clamping on and off.  ``agent.action.u`` and the holonomic force / torque are bit-exact;
  the bad-action flag equals the reference's assertion (any NaN, or |clamp(v)| > r) — a NaN must be flagged and
  kept with clamping on, as torch.clamp keeps it.
* Discrete and multi-discrete indices: bit-exact against the fp32 chain, within the float64 bound, exact at the
  special points; out-of-range indices flagged.
* DiffDrive, KinematicBicycle and Drone, RK4 and Euler: within 4x the first-order fp32 error bound of the float64
  reference, a bound tight enough that a plausible mistake in the model falls outside it.

libm's sin / cos / tan / atan2 are not CUDA's; the bound covers both.
"""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest
import torch

import action_cases as cases
import action_ref as ref
import vectorizedmultiagentsimulator_b200 as b200
from oracle.backend import use_oracle
from vectorizedmultiagentsimulator_b200 import _native as N

HERE = os.path.dirname(os.path.abspath(__file__))
SIM_DIR = os.path.join(HERE, "hostsim")
SIM_LIB = os.path.join(SIM_DIR, "_ingest.so")


def _build():
    sources = [os.path.join(SIM_DIR, "ingest.cpp"), os.path.join(SIM_DIR, "shim", "cuda_runtime.h")] + N.HEADERS
    if os.path.exists(SIM_LIB) and all(os.path.getmtime(f) <= os.path.getmtime(SIM_LIB) for f in sources):
        return
    subprocess.run(
        ["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-DVMAS_HOSTSIM",
         "-I", os.path.join(SIM_DIR, "shim"), "-I", N.CSRC, "-I", N.INCLUDE,
         os.path.join(SIM_DIR, "ingest.cpp"), "-o", SIM_LIB],
        check=True,
    )


@pytest.fixture(scope="module")
def sim():
    _build()
    lib = C.CDLL(SIM_LIB)
    lib.hostsim_ingest.argtypes = [C.c_int, C.POINTER(N.AgentActionsC)] + [C.c_int] * 4 + [C.c_void_p] * 6 + [C.c_int, C.c_void_p, C.c_void_p]
    lib.hostsim_ingest.restype = C.c_int
    return lib


class World:
    """Host arrays of one ingest call: E entities = A agents (agent i is entity i)."""

    def __init__(self, B, A):
        self.B, self.A = B, A
        self.pos = np.zeros((B, A, 2), np.float32)
        self.vel = np.zeros((B, A, 2), np.float32)
        self.rot = np.zeros((B, A), np.float32)
        self.ang_vel = np.zeros((B, A), np.float32)
        self.force = np.full((B, A, 2), np.nan, np.float32)
        self.torque = np.full((B, A), np.nan, np.float32)
        self.steps = np.zeros(B, np.float32)
        self.keep = []


def _agent(actions, size, dyn, index, u_range, mult, kind=N.ACT_CONTINUOUS, nvec=(), params=(), state=None):
    c = N.AgentActionsC()
    c.actions = actions.ctypes.data
    c.action_size, c.agent_index, c.entity_index, c.dynamics = size, index, index, dyn
    for j in range(size):
        c.u_range[j], c.u_multiplier[j] = u_range[j], mult[j]
    for j, n in enumerate(nvec):
        c.nvec[j] = n
    for j, p in enumerate(params):
        c.dyn_params[j] = p
    c.action_kind = kind
    c.dyn_state = None if state is None else state.ctypes.data
    return c


def _run(sim, w, agents, clamp, kin=False):
    """One ingest call; returns the bad-action flag."""
    arr = (N.AgentActionsC * len(agents))(*agents)
    flag = np.zeros(1, np.uint8)
    rc = sim.hostsim_ingest(
        int(kin), arr, len(agents), w.B, w.A, w.A, w.pos.ctypes.data, w.vel.ctypes.data, w.rot.ctypes.data,
        w.ang_vel.ctypes.data, w.force.ctypes.data, w.torque.ctypes.data, int(clamp), flag.ctypes.data, w.steps.ctypes.data,
    )
    assert rc == 0
    return bool(flag[0])


def assert_bits(got, want, what):
    """Same NaN positions, then the same bits everywhere else (torch.equal / == treat NaN as unequal)."""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    assert got.shape == want.shape, what
    assert np.array_equal(np.isnan(got), np.isnan(want)), f"{what}: NaN positions"
    ok = ~np.isnan(want)
    assert np.array_equal(got[ok].view(np.uint32), want[ok].view(np.uint32)), f"{what}: bits"


def _continuous_call(sim, layouts, actions, clamp, kin=False):
    """Every layout as one holonomic(-with-rotation) agent; returns (flag, world, u per agent)."""
    B = actions[0].shape[0]
    w = World(B, len(layouts))
    us, agents = [], []
    for i, ((r, m), a) in enumerate(zip(layouts, actions)):
        u = np.full(a.shape, np.nan, np.float32)
        us.append(u)
        w.keep += [a, u]
        c = _agent(a, a.shape[1], N.DYN_HOLONOMIC_ROT, i, r, m)
        c.u = u.ctypes.data
        agents.append(c)
    return _run(sim, w, agents, clamp, kin), w, us


@pytest.mark.parametrize("kin", [False, True])
@pytest.mark.parametrize("clamp", [False, True])
def test_continuous_edges_decode_bit_exact_and_flag_like_the_reference(sim, clamp, kin):
    rng = np.random.default_rng(1)
    layouts = cases.agent_layouts()
    B = 37
    legal = [cases.legal_batch(r, clamp, B, rng) for r, _ in layouts]
    flag, w, us = _continuous_call(sim, layouts, legal, clamp, kin)
    assert not flag, "a legal batch (every edge value at or inside the range) was flagged"
    assert np.array_equal(w.steps, np.ones(B, np.float32)), "the step counter advances once per env"
    for i, ((r, m), a, u) in enumerate(zip(layouts, legal, us)):
        want, flagged = ref.continuous(a, r, m, clamp)
        assert not flagged.any()
        assert_bits(u, want, f"agent {i} u")
        force, torque = ref.holonomic(want)
        assert_bits(w.force[:, i], force, f"agent {i} force")
        assert_bits(w.torque[:, i], torque, f"agent {i} torque")
    # each bad value alone, in the first and in the last env
    for i, (r_vec, m_vec) in enumerate(layouts):
        for j, r in enumerate(r_vec):
            for v in cases.edge_values(r)[1] + cases.edge_values(r)[2]:
                for env in (0, B - 1):
                    acts = [a.copy() for a in legal]
                    acts[i][env, j] = v
                    flag, w, us = _continuous_call(sim, layouts, acts, clamp, kin)
                    want, flagged = ref.continuous(acts[i], r_vec, m_vec, clamp)
                    assert flag == bool(flagged.any()), f"agent {i} component {j} value {v} env {env} clamp {clamp}"
                    assert_bits(us[i], want, f"agent {i} component {j} value {v}")
                    assert_bits(w.force[:, i], want[:, :2], f"agent {i} force, value {v}")
                    if math.isnan(v):
                        assert flag and np.isnan(us[i][env, j]), "NaN must be flagged and kept, clamped or not"


@pytest.mark.parametrize("nvec,multi", [([n], False) for n in cases.DISCRETE_N] + [([5, cases.BIG_N], True)]
                         + [(nv, m) for nv in cases.MULTI_NVEC for m in (False, True)])
def test_discrete_indices_decode_to_the_fp32_chain(sim, nvec, multi):
    r = [0.7, 3.0, 1.0][: len(nvec)]
    m = [0.7, 0.01, 1.0][: len(nvec)]
    if multi:
        per = [cases.discrete_indices(n) for n in nvec]
        B = max(len(p) for p in per)
        idx = np.stack([np.resize(p, B) for p in per], -1).astype(np.int64)
        actions = idx.copy()
    else:
        total = math.prod(nvec)
        flat = list(range(total)) if total <= 64 else sorted(set(
            k * (total // nvec[0]) + o for k in cases.discrete_indices(nvec[0]) for o in (0, total // nvec[0] - 1)))
        actions = np.array(flat, np.int64)[:, None]
        idx = ref.unravel(actions, nvec)
    B = actions.shape[0]
    w = World(B, 1)
    u = np.full((B, len(nvec)), np.nan, np.float32)
    c = _agent(actions, len(nvec), N.DYN_NONE, 0, r, m, N.ACT_MULTIDISCRETE if multi else N.ACT_DISCRETE, nvec)
    c.u = u.ctypes.data
    assert not _run(sim, w, [c], False)
    want, chain, flagged = ref.discrete(idx, nvec, r, m)
    assert not flagged.any()
    assert_bits(u, chain, "decoded vs the fp32 chain")
    assert np.all(np.abs(u - want.v) <= want.e), "decoded vs float64"
    k = np.asarray(idx)
    for j, n in enumerate(nvec):
        lo, hi = np.float32(-np.float32(r[j]) * np.float32(m[j])), np.float32(np.float32(r[j]) * np.float32(m[j]))
        lowest = (k[:, j] == (1 if n % 2 else 0))
        assert np.all(u[lowest, j] == lo) and np.all(u[k[:, j] == n - 1, j] == hi)
        if n % 2:
            zero = u[k[:, j] == 0, j]
            assert np.all(zero.view(np.uint32) == 0), "index 0 of an odd n is +0.0"
    # out of range: flagged
    for bad in ([-1, math.prod(nvec), 2 ** 40] if not multi else [-1, nvec[-1]]):
        a = actions.copy()
        if multi:
            a[B - 1, -1] = bad
        else:
            a[B - 1, 0] = bad
            assert ref.unravel(a, nvec)[B - 1].tolist() and (
                (ref.unravel(a, nvec)[B - 1] < 0) | (ref.unravel(a, nvec)[B - 1] >= nvec)).any()
        c.actions = a.ctypes.data
        assert _run(sim, World(B, 1), [c], False), f"index {bad} of nvec {nvec} not flagged"


# ---- kinematic models ---------------------------------------------------------------------------------------------
def _kin_ref(kind, u, rot, pos, vel, ang_vel, state, dt, rk4, **mistake):
    size, u_range, agent_kw, model_kw = cases.KIN[kind]
    mass, inertia = agent_kw["mass"], _inertia(kind)
    if kind == "diff":
        return None, None, *ref.diff_drive(u, rot, vel, ang_vel, dt, mass, inertia, rk4, **mistake)
    if kind == "bicycle":
        return None, None, *ref.bicycle(u, rot, vel, ang_vel, dt, mass, inertia, rk4, model_kw["l_f"], model_kw["l_r"],
                                        model_kw["max_steering_angle"], **mistake)
    I = (model_kw["I_xx"], model_kw["I_yy"], model_kw["I_zz"])
    return ref.drone(u, rot, pos, vel, ang_vel, state, dt, mass, inertia, rk4, I, **mistake)


def _inertia(kind):
    # the moment of inertia of the agents of action_cases.make_scenario: a sphere of radius 0.05 (core.py)
    return 0.5 * cases.KIN[kind][2]["mass"] * 0.05 ** 2


def _kin_params(kind, dt, rk4):
    size, u_range, agent_kw, model_kw = cases.KIN[kind]
    p = [dt, agent_kw["mass"], _inertia(kind), 1.0 if rk4 else 0.0]
    if kind == "bicycle":
        p += [model_kw["l_f"], model_kw["l_r"], model_kw["max_steering_angle"]]
    elif kind == "drone":
        p += [model_kw["I_xx"], model_kw["I_yy"], model_kw["I_zz"], 9.81]
    return p


def kinematic_inputs(kind, dt, rk4, seed=5):
    """(u, rot, pos, vel, ang_vel, drone state): half the envs with velocities equal to the commanded pose change."""
    rng = np.random.default_rng(seed)
    u, rot, ang_vel, state = cases.kinematic_cases(kind, rng, cases.KIN[kind][1])
    B = u.shape[0]
    pos = ((rng.random((B, 2)) * 2 - 1)).astype(np.float32)
    vel = ((rng.random((B, 2)) * 2 - 1) * 0.5).astype(np.float32)
    _, _, fx, fy, tq = _kin_ref(kind, u, rot, pos, np.zeros_like(vel), np.zeros_like(ang_vel), state, dt, rk4)
    mass, inertia = cases.KIN[kind][2]["mass"], _inertia(kind)
    cancel = np.arange(B) % 2 == 1  # v = delta / dt: the back-solve subtracts two nearly equal numbers
    vel[cancel, 0] = (fx.v * dt / mass)[cancel]
    vel[cancel, 1] = (fy.v * dt / mass)[cancel]
    ang_vel[cancel] = (tq.v * dt / inertia)[cancel]
    return u, rot, pos, vel, ang_vel, state


def _within(got, want, what, k=4.0):
    got = np.asarray(got, np.float64)
    err = np.abs(got - want.v)
    bad = ~(err <= k * want.e)
    assert not bad.any(), f"{what}: {int(bad.sum())} outside {k}x the bound, worst |err| / bound {np.max(err / np.maximum(want.e, 1e-300))}"


def _sim_kinematic(sim, kind, dt, rk4, inputs, clamp=False):
    u, rot, pos, vel, ang_vel, state = inputs
    B = u.shape[0]
    size, u_range, _, _ = cases.KIN[kind]
    w = World(B, 1)
    w.pos[:, 0], w.vel[:, 0], w.rot[:, 0], w.ang_vel[:, 0] = pos, vel, rot, ang_vel
    out_u = np.full(u.shape, np.nan, np.float32)
    ds = None if state is None else state.copy()
    dyn = dict(diff=N.DYN_DIFF_DRIVE, bicycle=N.DYN_BICYCLE, drone=N.DYN_DRONE)[kind]
    c = _agent(u, size, dyn, 0, [1e30] * size, [1.0] * size, params=_kin_params(kind, dt, rk4), state=ds)
    c.u = out_u.ctypes.data
    assert not _run(sim, w, [c], clamp, kin=True)
    return out_u, w.force[:, 0], w.torque[:, 0], ds


MISTAKES = {
    "diff": [dict(euler=True), dict(dt2=True)],
    "bicycle": [dict(euler=True), dict(no_steer_clamp=True), dict(no_slip=True), dict(dt2=True)],
    "drone": [dict(euler=True), dict(no_thrust_offset=True), dict(yaw_not_from_rot=True), dict(dt2=True)],
}


@pytest.mark.parametrize("dt", cases.DTS)
@pytest.mark.parametrize("kind", ["diff", "bicycle", "drone"])
def test_kinematic_models_within_the_fp32_bound_of_float64(sim, kind, dt):
    ratios, caught = [], {i: False for i in range(len(MISTAKES[kind]))}
    for rk4 in (True, False):
        inputs = kinematic_inputs(kind, dt, rk4)
        u, rot, pos, vel, ang_vel, state = inputs
        got_u, fxy, tq, ds = _sim_kinematic(sim, kind, dt, rk4, inputs)
        u_out, new_state, fx, fy, t = _kin_ref(kind, u, rot, pos, vel, ang_vel, state, dt, rk4)
        what = f"{kind} dt={dt} rk4={rk4}"
        _within(fxy[:, 0], fx, what + " force x")
        _within(fxy[:, 1], fy, what + " force y")
        _within(tq, t, what + " torque")
        if kind == "drone":
            _within(got_u, u_out, what + " u (thrust offset in place)")
            _within(ds, new_state, what + " drone state")
        else:
            assert_bits(got_u, u, what + " u")
        for r in (fx, fy, t):  # (the odd envs cancel on purpose: there |ref| ~ 0 and the ratio means nothing)
            r = r[::2]
            nz = np.abs(r.v) > 0
            ratios.append(r.e[nz] / np.abs(r.v[nz]))
        # each plausible mistake lands outside the tolerance somewhere
        for i, mistake in enumerate(MISTAKES[kind]):
            if mistake.get("euler") and not rk4:
                continue
            _, _, mfx, mfy, mt = _kin_ref(kind, u, rot, pos, vel, ang_vel, state, dt, rk4, **mistake)
            for g, m in ((fxy[:, 0], mfx), (fxy[:, 1], mfy), (tq, mt)):
                caught[i] |= bool((np.abs(g - m.v) > 4 * m.e).any())
    assert all(caught.values()), f"{kind}: mistakes inside the tolerance: {[MISTAKES[kind][i] for i, c in caught.items() if not c]}"
    assert np.median(np.concatenate(ratios)) < 1e-5, "the bound is too loose to tell a wrong model from a right one"


# ---- the torch host path (CPU oracle env) -------------------------------------------------------------------------
def _oracle_env(agents, clamp, dt=0.1, B=37):
    with use_oracle():
        return b200.make_env(cases.make_scenario(agents, dt), num_envs=B, device="cpu", seed=0, clamp_actions=clamp,
                             action_checks="sync")


@pytest.mark.parametrize("clamp", [False, True])
def test_host_path_decodes_and_flags_like_the_reference(clamp):
    layouts = cases.agent_layouts()
    env = _oracle_env([("holo_rot", r, m, None) for r, m in layouts], clamp)
    rng = np.random.default_rng(2)
    B = env.num_envs
    legal = [cases.legal_batch(r, clamp, B, rng) for r, _ in layouts]
    env._apply_actions([torch.from_numpy(a) for a in legal])  # no assertion: every value at or inside the range
    for i, ((r, m), a) in enumerate(zip(layouts, legal)):
        want, _ = ref.continuous(a, r, m, clamp)
        agent = env.agents[i]
        assert_bits(agent.action.u.numpy(), want, f"agent {i} u")
        assert_bits(agent.state.force.numpy(), want[:, :2], f"agent {i} force")
        assert_bits(agent.state.torque.numpy()[:, 0], want[:, 2], f"agent {i} torque")
    i, (r_vec, m_vec) = 3, layouts[3]
    for j, r in enumerate(r_vec[:4]):
        for v in cases.edge_values(r)[1] + cases.edge_values(r)[2]:
            acts = [a.copy() for a in legal]
            acts[i][B - 1, j] = v
            _, flagged = ref.continuous(acts[i], r_vec, m_vec, clamp)
            if flagged.any():
                with pytest.raises(AssertionError):
                    env._apply_actions([torch.from_numpy(a) for a in acts])
            else:
                env._apply_actions([torch.from_numpy(a) for a in acts])


@pytest.mark.parametrize("dt", cases.DTS)
@pytest.mark.parametrize("kind", ["diff", "bicycle", "drone"])
def test_host_path_kinematic_models_within_the_fp32_bound(kind, dt):
    for rk4 in (True, False):
        inputs = kinematic_inputs(kind, dt, rk4)
        u, rot, pos, vel, ang_vel, state = inputs
        B = u.shape[0]
        size, u_range, agent_kw, model_kw = cases.KIN[kind]
        extra = (agent_kw, model_kw, "rk4" if rk4 else "euler")
        env = _oracle_env([(kind, [1e30] * size, [1.0] * size, extra)], False, dt, B)
        agent = env.agents[0]
        agent.set_pos(torch.from_numpy(pos), batch_index=None)
        agent.set_vel(torch.from_numpy(vel), batch_index=None)
        agent.set_rot(torch.from_numpy(rot)[:, None], batch_index=None)
        agent.set_ang_vel(torch.from_numpy(ang_vel)[:, None], batch_index=None)
        if state is not None:
            agent.dynamics.drone_state = torch.from_numpy(state.copy())
        env._apply_actions([torch.from_numpy(u)])
        u_out, new_state, fx, fy, t = _kin_ref(kind, u, rot, pos, vel, ang_vel, state, dt, rk4)
        what = f"host {kind} dt={dt} rk4={rk4}"
        _within(agent.state.force[:, 0].numpy(), fx, what + " force x")
        _within(agent.state.force[:, 1].numpy(), fy, what + " force y")
        _within(agent.state.torque[:, 0].numpy(), t, what + " torque")
        if kind == "drone":
            _within(agent.action.u.numpy(), u_out, what + " u")
            _within(agent.dynamics.drone_state.numpy(), new_state, what + " drone state")
