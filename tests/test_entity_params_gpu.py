"""Per-env entity mass and friction coefficients on the GPU: the generic and the run-time specialised kernels
against the reference's recorded roll-out of ``crafted_randomised`` (teacher-forced), bit-equality between the
kernels, per-env gravity on the specialised kernel (wind_flocking), and a captured CUDA graph that keeps
reading re-drawn values."""
import os

import pytest
import torch

import crafted_params
import golden_pack
from golden_util import GOLDEN_DIR, STATE_KEYS, load, teacher_forced_steps
from vectorizedmultiagentsimulator_b200 import _native, codegen, jit
from vectorizedmultiagentsimulator_b200.simulator import plan as P

pytestmark = pytest.mark.gpu

FIXTURE = os.path.join(GOLDEN_DIR, "reference", "teacher_forced", "crafted_randomised-0.npz")
STATE = ("pos", "vel", "rot", "ang_vel")
COLS = {"mass": P.EP_MASS, "linear_friction": P.EP_LIN_FRIC, "angular_friction": P.EP_ANG_FRIC}


class _Slab:
    def __init__(self, state, device):
        self.t = {k: state[k].to(device).contiguous() for k in STATE_KEYS}

    def tensors(self):
        return tuple(self.t[k] for k in STATE_KEYS)


def _tables(tables, device, mapping, entry):
    dt = _native.DeviceTables(tables, None, device, mapping=mapping)
    for k, v in entry["fixed_rot"].items():
        dt.joint_rot[:, k] = v.reshape(-1).to(device)
    for e, g in entry["ent_gravity"].items():
        dt.ent_gravity[:, e] = g.to(device)
    for e, values in entry["ent_params"].items():
        for attr, v in values.items():
            if attr in COLS:
                dt.ent_params[:, e, COLS[attr]] = v.reshape(-1).to(device)
    return dt


def _specialise(desc):
    if not jit.available():
        pytest.skip("no nvcc / JIT switched off")
    job = jit.request(desc)
    assert job is not None, "the world must be specialisable"
    assert job.done.wait(timeout=600) and job.error is None, job.error
    return job


def test_three_kernels_match_reference_and_each_other():
    rec = golden_pack.load(FIXTURE)
    desc = P.WorldDescription.from_json(rec["desc"])
    tables = P.build_tables(desc)
    device, lib = torch.device("cuda:0"), _native.load()
    job = _specialise(desc)
    assert lib.vmas_b200_find_specialization(codegen.world_hash(desc)) == job.index
    prev = None
    for t, entry in enumerate(rec["steps"]):
        state = {k: v.clone() for k, v in entry.get("state_in", prev).items() if k in STATE}
        state["force"], state["torque"] = entry["force"].clone(), entry["torque"].clone()
        outs = {}
        for mapping in ("thread_per_env", "lanes_per_env", "specialized"):
            dt = _tables(tables, device, mapping, entry)
            assert dt.mapping == mapping and dt.ent_params is not None
            if mapping == "specialized":
                assert dt.specialization >= 0
            slab = _Slab(state, device)
            _native.world_step(lib, dt, slab)
            outs[mapping] = slab
        for k in STATE:
            want = entry["out"][k]
            got = outs["thread_per_env"].t[k].cpu()
            err = (got - want).abs()
            assert bool((err <= 1e-5 + 1e-4 * want.abs()).all()), f"step {t} {k}: max |diff| {float(err.max())}"
        for k in STATE_KEYS:
            base = outs["thread_per_env"].t[k]
            assert torch.equal(base, outs["lanes_per_env"].t[k]), f"step {t} {k}: lanes_per_env"
            assert torch.equal(base, outs["specialized"].t[k]), f"step {t} {k}: specialized"
        prev = entry["out"]


def test_specialised_kernel_needs_its_parameter_table():
    rec = golden_pack.load(FIXTURE)
    desc = P.WorldDescription.from_json(rec["desc"])
    tables = P.build_tables(desc)
    _specialise(desc)
    device, lib = torch.device("cuda:0"), _native.load()
    entry = rec["steps"][0]
    dt = _tables(tables, device, "specialized", entry)
    slab = _Slab({**entry["state_in"], "force": entry["force"], "torque": entry["torque"]}, device)
    st = dt.state_struct(slab)
    import ctypes as C

    rc = lib.vmas_b200_world_step(C.byref(dt.cfg), C.byref(dt.tb), C.byref(st), dt.mask.data_ptr(), 1,
                                  _native._stream(device))
    assert rc < 0 and b"invalid" in lib.vmas_b200_last_error().lower()


def test_wind_flocking_specialised_equals_generic():
    fix, desc, tables = load("wind_flocking")
    device, lib = torch.device("cuda:0"), _native.load()
    _specialise(desc)
    for t, state_in, fixed_rot, _ in teacher_forced_steps(fix):
        outs = []
        for mapping in ("thread_per_env", "specialized"):
            dt = _native.DeviceTables(tables, None, device, mapping=mapping)
            assert dt.mapping == mapping
            for e, g in state_in["ent_gravity"].items():
                dt.ent_gravity[:, e] = g.to(device)
            slab = _Slab(state_in, device)
            _native.world_step(lib, dt, slab)
            outs.append(slab)
        for k in STATE_KEYS:
            assert torch.equal(outs[0].t[k], outs[1].t[k]), f"step {t} {k}"


class _Quiet:
    """crafted_params' world without its own re-draws: the test changes the values between steps."""

    def __new__(cls):
        sc = crafted_params.make_scenario("vectorizedmultiagentsimulator_b200")
        type(sc).pre_step = lambda self: None
        return sc


def _redraw(env, t, gen):
    """Half the envs: in place on odd t, by assigning a fresh tensor on even t (gravity: always in place)."""
    world = env.world
    n = world.batch_dim
    envs = (torch.arange(n) % 2 == t % 2).to(world.device)
    for e in world.entities:
        for attr in crafted_params.PER_ENV.get(e.name, ()):
            new = (torch.rand(n, 2 if attr == "gravity" else 1, generator=gen) * 0.5 + 0.5).to(world.device)
            cur = getattr(e, attr)
            if t % 2 or attr == "gravity":  # (a new Entity.gravity tensor is a new address: edited in place)
                cur[envs] = new[envs]
            else:
                setattr(e, attr, torch.where(envs.unsqueeze(-1), new, cur))


def test_cuda_graph_rereads_redrawn_parameters():
    import vectorizedmultiagentsimulator_b200 as b200

    if not jit.available():
        pytest.skip("no nvcc / JIT switched off")
    n = 256
    envs = [b200.make_env(_Quiet(), num_envs=n, device="cuda:0", seed=0, cuda_graph=g) for g in (False, True)]
    captures = []
    graphed = envs[1]
    real_capture = graphed._capture
    graphed._capture = lambda *a, **k: (captures.append(1), real_capture(*a, **k))[1]
    for env in envs:
        env.reset(seed=1)
        env.world._get_backend().wait_for_jit()
    assert envs[1].world._get_backend()._dev_tables.specialization >= 0
    gens = [torch.Generator().manual_seed(7) for _ in envs]
    act_gen = torch.Generator().manual_seed(3)
    versions = None
    requests = None
    for t in range(20):
        actions = [(torch.rand(n, a.action_size, generator=act_gen) * 2 - 1).cuda() for a in envs[0].agents]
        outs = []
        for env, gen in zip(envs, gens):
            _redraw(env, t, gen)
            outs.append(env.step([a.clone() for a in actions]))
        for a, b in zip(outs[0][0], outs[1][0]):
            assert torch.equal(a, b), f"step {t}: observations"
        for e0, e1 in zip(envs[0].world.entities, envs[1].world.entities):
            assert torch.equal(e0.state.pos, e1.state.pos) and torch.equal(e0.state.vel, e1.state.vel), f"step {t}"
        if t == 3:
            versions = [env.world._plan_version for env in envs]
            requests = len(jit._jobs)
    assert [env.world._plan_version for env in envs] == versions
    assert len(jit._jobs) == requests
    assert len(captures) == 1 and graphed.graph_replays >= 15
