"""The block-per-env step kernel on the GPU, and worlds past the thread-per-env kernel's limit.

* ``block_per_env`` equals ``thread_per_env`` bit for bit on every golden world and on the per-env-parameter
  world: whole steps with and without the batch-wide broad phase, a batch that leaves the thread-per-env
  kernel a partial last block, and ``batch_dim = 1``.
* The three large crafted worlds (160, 520 and 1024 entities) against the reference's recorded roll-outs,
  teacher-forced, within ``1e-5 + 1e-4|x|`` widened by the joint envelope of DESIGN.md section 6.
* A shipped scenario past the old limit (flocking with 150 agents and its LIDAR observations) on CUDA
  against the same env on the CPU oracle: teacher-forced and in a 10-step roll-out, eager and CUDA-graph
  steps bit-identical, every spawn successful.
* At 1024 entities the observation gather and ``post_step`` equal the ``torch.cat`` formulation bit for bit.
"""
import os

import pytest
import torch

import golden_pack
import vectorizedmultiagentsimulator_b200 as b200
from envutil import flatten, sync_env
from golden_util import GOLDEN_DIR, STATE_KEYS, golden_names, load, same_result, teacher_forced_steps
from oracle.backend import use_oracle
from test_large_world import COLS, LARGE, load_large, ulp_sensitivity
from vectorizedmultiagentsimulator_b200 import _native
from vectorizedmultiagentsimulator_b200.simulator import plan as P

pytestmark = pytest.mark.gpu

DEVICE = torch.device("cuda:0")
STATE = ("pos", "vel", "rot", "ang_vel")


class _Slab:
    def __init__(self, state, device, n=None):
        self.t = {k: state[k][:n].to(device).contiguous() for k in STATE_KEYS}

    def tensors(self):
        return tuple(self.t[k] for k in STATE_KEYS)


def _tables(tables, mapping, fixed_rot=None, ent_gravity=None, ent_params=None):
    dt = _native.DeviceTables(tables, None, DEVICE, mapping=mapping)
    assert dt.mapping == mapping
    for k, v in (fixed_rot or {}).items():
        dt.joint_rot[:, k] = v.reshape(-1).to(DEVICE)
    for e, g in (ent_gravity or {}).items():
        dt.ent_gravity[:, e] = g.to(DEVICE)
    for e, values in (ent_params or {}).items():
        for attr, v in values.items():
            if attr in COLS:
                dt.ent_params[:, e, COLS[attr]] = v.reshape(-1).to(DEVICE)
    return dt


def _worlds():
    for name in golden_names():
        fix, _, tables = load(name)
        yield name, tables, [(t, s, fr, s.get("ent_gravity"), None) for t, s, fr, _ in teacher_forced_steps(fix)]
    rec = golden_pack.load(os.path.join(GOLDEN_DIR, "reference", "teacher_forced", "crafted_randomised-0.npz"))
    tables = P.build_tables(P.WorldDescription.from_json(rec["desc"]))
    yield "crafted_randomised", tables, [
        (t, s, fr, e["ent_gravity"], e["ent_params"]) for (t, s, fr, _), e in zip(teacher_forced_steps(rec), rec["steps"])
    ]


WORLDS = list(_worlds())


@pytest.mark.parametrize("i", range(len(WORLDS)), ids=[w[0] for w in WORLDS])
def test_block_per_env_equals_thread_per_env_bitwise(i):
    name, tables, steps = WORLDS[i]
    lib = _native.load()
    B = steps[0][1]["pos"].shape[0]
    # all envs; a batch the thread-per-env kernel's 64- and 32-env blocks do not divide; one env
    sizes = sorted({B, min(B, 37), 1}, reverse=True)
    checked = 0
    for t, state_in, fixed_rot, ent_gravity, ent_params in steps:
        if t % 3:
            continue
        for n in sizes:
            for exact in (True, False):
                outs = []
                for mapping in ("thread_per_env", "block_per_env"):
                    dt = _tables(tables, mapping, fixed_rot, ent_gravity, ent_params)
                    dt.cfg.batch_dim = n
                    slab = _Slab(state_in, DEVICE, n)
                    _native.world_step(lib, dt, slab, exact_broad_phase=exact)
                    outs.append(slab)
                for k in STATE_KEYS:
                    assert same_result(outs[1].t[k], outs[0].t[k]), f"{name} step {t} B={n} broad phase {exact}: {k}"
                checked += 1
    torch.cuda.synchronize()
    assert checked >= 4


@pytest.mark.parametrize("case", LARGE)
def test_large_world_vs_reference(case):
    rec, desc, tables = load_large(case)
    lib = _native.load()
    worst = 0.0
    for t, state_in, fixed_rot, want in teacher_forced_steps(rec):
        dt = _native.DeviceTables(tables, None, DEVICE)  # auto: the block-per-env kernel
        assert dt.mapping == "block_per_env"
        for k, v in fixed_rot.items():
            dt.joint_rot[:, k] = v.reshape(-1).to(DEVICE)
        slab = _Slab(state_in, DEVICE)
        assert _native.world_step(lib, dt, slab) >= 1
        sens = ulp_sensitivity(tables, state_in, fixed_rot)
        for k in STATE_KEYS:
            err = (slab.t[k].cpu() - want[k]).abs()
            atol = 1e-5 + 4.0 * sens[k]
            assert bool((err <= atol + 1e-4 * want[k].abs()).all()), f"{case} step {t} {k}: max |err| {float(err.max())}"
            worst = max(worst, float(err.max()))
    print(f"{case}: max |err| vs reference {worst:.3e}")


def _compare(got, want, what, atol, rtol=1e-4):
    g, w = flatten(got), flatten(want)
    assert len(g) == len(w), what
    for a, b in zip(g, w):
        a = a.cpu()
        assert a.shape == b.shape and a.dtype == b.dtype, what
        if a.dtype == torch.bool:
            assert torch.equal(a, b), what
        else:
            err = (a - b).abs()
            assert bool((err <= atol + rtol * b.abs()).all()), f"{what}: max |err| {float(err.max())}"


def _same_outputs(a, b, what):
    for x, y in zip(flatten(a), flatten(b)):
        assert same_result(x, y, atol=2e-4), what


def test_flocking_with_150_agents_on_cuda():
    n_envs = 24
    kwargs = dict(n_agents=150, min_dist_between_entities=0.1)
    with use_oracle():
        cpu = b200.make_env("flocking", num_envs=n_envs, device="cpu", seed=0, **kwargs)
    eager = b200.make_env("flocking", num_envs=n_envs, device="cuda", seed=0, **kwargs)
    graph = b200.make_env("flocking", num_envs=n_envs, device="cuda", seed=0, cuda_graph=True, **kwargs)
    assert len(eager.world.entities) == 156
    for env in (eager, graph):
        env.reset()
        assert env.world.spawn_failures() == 0
    gen = torch.Generator().manual_seed(5)

    def actions():
        return [(torch.rand(n_envs, a.action_size, generator=gen) * 2 - 1) * a.action.u_range_tensor for a in cpu.agents]

    for t in range(5):  # teacher-forced (the graph is captured on the third step and replayed after)
        sync_env(cpu, eager)
        sync_env(cpu, graph)
        act = actions()
        want = cpu.step([a.clone() for a in act])
        got = eager.step([a.to("cuda") for a in act])
        again = graph.step([a.to("cuda") for a in act])
        _compare(got[0], want[0], f"step {t} obs", atol=1e-5)
        _compare(got[1], want[1], f"step {t} rews", atol=2e-4)
        _compare(got[2], want[2], f"step {t} dones", atol=0)
        _same_outputs(again, got, f"step {t}: graph vs eager")
    assert eager.world._get_backend()._dev_tables.mapping == "block_per_env"
    sync_env(cpu, eager)
    sync_env(cpu, graph)
    for t in range(10):  # free roll-out
        act = actions()
        want = cpu.step([a.clone() for a in act])
        got = eager.step([a.to("cuda") for a in act])
        again = graph.step([a.to("cuda") for a in act])
        _same_outputs(again, got, f"roll-out step {t}: graph vs eager")
    _compare(got[0], want[0], "roll-out obs", atol=1e-4)
    assert graph.graph_replays >= 10
    eager.check_actions_now()


def test_observations_of_1024_entities_equal_torch_cat():
    rec, desc, tables = load_large("large_1024-2")
    assert desc.n_entities == 1024
    lib = _native.load()
    N = _native
    dt = _native.DeviceTables(tables, None, DEVICE)
    slab = _Slab(rec["steps"][-1]["out"], DEVICE)
    pos, vel, rot, ang_vel = (slab.t[k] for k in STATE)
    B, E = pos.shape[0], pos.shape[1]
    table, want = [], []
    for e, other in ((0, E - 1), (E - 1, 511), (700, 3)):  # rows from both ends of the staged slab
        cols, parts = [], []
        for k in range(2):
            cols.append((N.OBS_COPY, (N.OBS_POS << 24) | (2 * e + k), 0, 0))
        parts.append(pos[:, e])
        for k in range(2):
            cols.append((N.OBS_DIFF, (N.OBS_VEL << 24) | (2 * e + k), (N.OBS_VEL << 24) | (2 * other + k), 0))
        parts.append(vel[:, e] - vel[:, other])
        for k in range(2):
            cols.append((N.OBS_DIFF, (N.OBS_POS << 24) | (2 * other + k), (N.OBS_POS << 24) | (2 * e + k), 0))
        parts.append(pos[:, other] - pos[:, e])
        cols.append((N.OBS_COPY, (N.OBS_ANG_VEL << 24) | e, 0, 0))
        parts.append(ang_vel[:, e:e + 1])
        bits = torch.tensor(torch.pi, dtype=torch.float32).view(torch.int32).item()
        cols.append((N.OBS_REMAINDER, (N.OBS_ROT << 24) | other, 0, bits))
        parts.append(rot[:, other:other + 1] % torch.pi)
        table.append(cols)
        want.append(torch.cat(parts, dim=-1))
    want = torch.stack(want)
    rows, width = want.shape[0], want.shape[-1]
    columns = torch.tensor(table, dtype=torch.int32, device=DEVICE).contiguous()
    out = torch.full((rows, B, width), -7.0, device=DEVICE)
    _native.gather_observations(lib, dt, slab, columns, rows, width, out)
    assert torch.equal(out, want)
    out2 = torch.full((rows, B, width), -7.0, device=DEVICE)
    _native.post_step(lib, dt, slab, None, columns, rows, width, out2)
    assert torch.equal(out2, want)
