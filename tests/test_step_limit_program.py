"""The step limit of a bounded episode (``max_steps``, ``terminated_truncated``) as a step program, on the CPU.

On CUDA, ``Environment._done`` runs ``_limit_program`` in place of its torch statements when the scenario's
``done()`` is an output of this step's program, and a captured step splices that program into the scenario's
(``splice_program``) so that the whole-step kernel computes it too.  Checked here:

* the limit program, interpreted by the oracle, equals ``steps >= max_steps`` and ``terminated + truncated`` bit for
  bit: counters below, at and past the limit, ``max_steps = 0``, and a counter of 2^24 against 2^24 + 1 (torch
  compares an fp32 counter with the limit rounded to fp32, and so does the program's constant);
* the splice: registers and buffer slots numbered on from the scenario's, ``terminated`` read from the register the
  scenario's program stores it from, the counter read by ``OP_STEP_COUNT``; the merged program gives what the two
  programs give one after the other (balance and transport);
* the epilogue of the whole-step kernel (``spec_epilogue`` in csrc/spec_kernel.cuh, compiled with g++ against the
  ``cuda_runtime.h`` stand-in of tests/hostsim) with ``OP_STEP_COUNT`` driven by a given count, one lane per env and
  on a lane pair, against the oracle's interpretation; the counter's buffer is poisoned so that only the count handed
  to the epilogue can make it right.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

import vectorizedmultiagentsimulator_b200 as b200
from oracle.backend import use_oracle
from vectorizedmultiagentsimulator_b200 import _native, codegen
from vectorizedmultiagentsimulator_b200.simulator import plan as P
from vectorizedmultiagentsimulator_b200.simulator import program as SP
from vectorizedmultiagentsimulator_b200.simulator.environment.environment import splice_program

HERE = os.path.dirname(os.path.abspath(__file__))
SIM_DIR = os.path.join(HERE, "hostsim")
SCENARIOS = [("balance", dict(n_agents=4)), ("transport", dict(n_agents=4))]
LIMITS = [(5, False), (5, True), (None, True)]  # (max_steps, terminated_truncated)


def _env(name, kwargs, max_steps, split, n_envs=16, steps=3):
    with use_oracle():
        env = b200.make_env(name, num_envs=n_envs, device="cpu", seed=0, max_steps=max_steps,
                            terminated_truncated=split, **kwargs)
        env.reset()
        torch.manual_seed(0)
        for _ in range(steps):
            env.step(env.get_random_actions())
    return env


def _torch_statements(env, terminated):
    """What ``Environment._done`` computes with torch ops: dones, or truncated."""
    truncated = env.steps >= env.max_steps if env.max_steps is not None else None
    if env.terminated_truncated:
        return torch.zeros_like(terminated) if truncated is None else truncated
    return terminated + truncated


@pytest.mark.parametrize("max_steps,split", [(7, False), (7, True), (0, False), (0, True), (None, True)])
def test_limit_program_equals_the_torch_statements(max_steps, split):
    env = _env("balance", dict(n_agents=3), max_steps, split, n_envs=12, steps=0)
    counts = torch.tensor([0, 1, 5, 6, 7, 8, 9, 100, 0, 7, 6, 2 ** 24], dtype=torch.float32)
    env.steps.copy_(counts)
    terminated = torch.tensor([False, True] * 6)
    with use_oracle():
        limit = env._limit_program()
        env._limit_input = terminated
        limit.run()
    want = _torch_statements(env, terminated)
    assert limit.out.tensor.dtype == want.dtype == torch.bool
    assert torch.equal(limit.out.tensor, want)


@pytest.mark.parametrize("split", [False, True])
def test_limit_constant_is_rounded_to_fp32_as_torch_rounds_it(split):
    env = _env("balance", dict(n_agents=3), 2 ** 24 + 1, split, n_envs=4, steps=0)
    env.steps.copy_(torch.tensor([2 ** 24 - 1, 2 ** 24, 2 ** 24 + 2, 0], dtype=torch.float32))
    terminated = torch.zeros(4, dtype=torch.bool)
    with use_oracle():
        limit = env._limit_program()
        env._limit_input = terminated
        limit.run()
    want = _torch_statements(env, terminated)
    assert want.tolist() == [False, True, True, False]  # (2^24 + 1 is 2^24 in fp32)
    assert torch.equal(limit.out.tensor, want)


def _programs(env):
    """(scenario program, its instructions with entity indices, limit program, merged instructions, registers,
    slot map, register of terminated)."""
    prog = env.scenario._step_program().finalize()
    index = {id(e): i for i, e in enumerate(env.world.entities)}
    instrs = prog.instructions(lambda e: index[id(e)])
    limit = env._limit_program()
    store_of = {b: a for op, _, a, b, _, _ in instrs if op in (SP.OP_STORE_F32, SP.OP_STORE_BOOL)}
    feed_reg = store_of[prog.out_done._slot] if limit.feed_slot is not None else None
    merged, n_regs, slots = splice_program(instrs, prog.n_regs, len(prog.buffers), limit.instructions(None),
                                           limit.feed_slot, feed_reg, limit.count_slot)
    return prog, instrs, limit, merged, n_regs, slots, feed_reg


@pytest.mark.parametrize("max_steps,split", LIMITS)
@pytest.mark.parametrize("name,kwargs", SCENARIOS)
def test_splice_maps_registers_slots_and_stores(name, kwargs, max_steps, split):
    env = _env(name, kwargs, max_steps, split)
    prog, instrs, limit, merged, n_regs, slots, feed_reg = _programs(env)
    n_slots = len(prog.buffers)
    assert merged[: len(instrs)] == instrs  # the scenario's program is left as it is
    extra = merged[len(instrs):]
    # every limit buffer but terminated gets a slot past the scenario's, in order of first use
    used = [j for j in range(len(limit.buffers)) if j != limit.feed_slot]
    assert sorted(slots) == used and sorted(slots.values()) == list(range(n_slots, n_slots + len(used)))
    # one instruction fewer where the load of terminated was dropped
    assert len(extra) == len(limit.instr) - (limit.feed_slot is not None)
    written = [dst for op, dst, *_ in extra if op not in (SP.OP_STORE_F32, SP.OP_STORE_BOOL)]
    assert written == list(range(prog.n_regs, n_regs)) and n_regs <= SP.MAX_REGS
    ops = [op for op, *_ in extra]
    assert ops.count(SP.OP_STEP_COUNT) == (max_steps is not None)
    assert SP.OP_LOAD_F32 not in ops and SP.OP_LOAD_BOOL not in ops
    for op, dst, a, b, arg, imm in extra:
        if op == SP.OP_STEP_COUNT:
            assert a == slots[limit.count_slot]
        if op == SP.OP_OR:  # terminated | (count >= max): terminated is the register the scenario stores dones from
            assert a == feed_reg
        if op == SP.OP_CONST and max_steps is not None:
            assert imm == float(max_steps)
    op, _, reg, slot, _, _ = extra[-1]
    assert op == SP.OP_STORE_BOOL and slot == slots[limit.out._slot] and reg == written[-1]


@pytest.mark.parametrize("max_steps,split", LIMITS)
@pytest.mark.parametrize("name,kwargs", SCENARIOS)
def test_merged_program_gives_what_the_two_programs_give(name, kwargs, max_steps, split):
    env = _env(name, kwargs, max_steps, split)
    prog, instrs, limit, merged, n_regs, slots, _ = _programs(env)
    env.steps.copy_(torch.arange(env.num_envs, dtype=torch.float32) % 9)
    carried = [prog.resolve(b).clone() for b in prog.buffers]  # (the shaping carry is overwritten by a run)
    # the two programs one after the other
    with use_oracle():
        prog.run()
        env._limit_input = prog.out_done.tensor
        limit.run()
    want = [prog.resolve(b).clone() for b in prog.buffers] + [limit.out.tensor.clone()]
    # the merged one, on a copy of the inputs: OP_STEP_COUNT is the load of the counter off the one-kernel step
    for b, t in zip(prog.buffers, carried):
        prog.resolve(b).copy_(t)
    one = SP.StepProgram(env.world)
    one.buffers = list(prog.buffers) + [None] * len(slots)
    for old, new in slots.items():
        one.buffers[new] = limit.buffers[old]
    one.instr = list(prog.instr)
    for op, dst, a, b, arg, imm in merged[len(instrs):]:
        one.instr.append((SP.OP_LOAD_F32 if op == SP.OP_STEP_COUNT else op, dst, a, b, arg, imm, None))
    limit.out.tensor.zero_()
    with use_oracle():
        env.world._get_backend().run_program(one)
    got = [prog.resolve(b) for b in prog.buffers] + [limit.out.tensor]
    for slot, (g, w) in enumerate(zip(got, want)):
        assert torch.equal(g, w), f"buffer {slot}"


SOURCE = """// GENERATED by tests/test_step_limit_program.py (test infrastructure)
#include "spec_kernel.cuh"
namespace vmas {{
{world}
{post}
}}
using namespace vmas;
using W = {name};
using Q = {post_name};
static_assert(epi_counts<Q>(), "the program reads the step counter");

// The epilogue of every env as step_env_kernel<W, Q, G> runs it, with the count its prologue hands over
// (counts == nullptr: EpiLoadCount, the load step_fused_kernel does); the lanes of a pair one after the other.
extern "C" int hostsim_epilogue(int G, int B, float* pos, float* vel, float* rot, float* ang_vel, float* force,
                                float* torque, const float* counts, void** buffers) {{
  SpecArgs a;
  a.st.pos = pos; a.st.vel = vel; a.st.rot = rot; a.st.ang_vel = ang_vel; a.st.force = force; a.st.torque = torque;
  a.joint_rot = nullptr; a.mask = nullptr; a.batch_dim = B; a.use_mask = 0; a.first_substep = 0; a.n_substeps = 1;
  a.order = nullptr; a.sig = nullptr;
  EpiArgs e;
  e.obs_out = nullptr;
  for (int i = 0; i < VMAS_PROG_MAX_BUFFERS; ++i) e.buffers[i] = buffers[i];
  constexpr int NA = W::A > 0 ? W::A : 1;
  for (long env = 0; env < B; ++env) {{
    SpecRows<W> rows;
    EnvRegs<W::E> r;
    float afx[NA], afy[NA], atq[NA];
    rows.load_pos_rot(a, env);
    rows.load_rest(a, env);
    rows.unpack_pos_rot(r);
    rows.unpack_rest(r, afx, afy, atq);
    if (!counts) {{
      spec_epilogue<W, Q>(r, a, e, env);
      continue;
    }}
    const float c = counts[env];
    const auto count = [c](const float*) {{ return c; }};
    if (G == 1) {{
      spec_epilogue<W, Q>(r, a, e, env, 1, 0, EpiOneLane{{}}, count);
    }} else {{
      float carry[8];
      int n0 = 0, n1 = 0;
      spec_epilogue<W, Q>(r, a, e, env, 2, 0, [&](float v) {{ return carry[n0++] = v; }}, count);
      spec_epilogue<W, Q>(r, a, e, env, 2, 1, [&](float) {{ return carry[n1++]; }}, count);
    }}
  }}
  return 0;
}}
"""


def _compile(desc, instrs, tag):
    name, text, _ = codegen.emit_world(desc, "hostsim")
    post_name, post_text, _ = codegen.emit_post(None, instrs)
    src = os.path.join(SIM_DIR, f"_fused_limit_{tag}.cpp")
    lib = os.path.join(SIM_DIR, f"_fused_limit_{tag}.so")
    with open(src, "w") as fh:
        fh.write(SOURCE.format(world=text, post=post_text, name=name, post_name=post_name))
    subprocess.run(
        ["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-DVMAS_HOSTSIM", "-x", "c++",
         "-I", os.path.join(SIM_DIR, "shim"), "-I", _native.CSRC, "-I", _native.INCLUDE, src, "-o", lib],
        check=True,
    )
    out = C.CDLL(lib)
    out.hostsim_epilogue.argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 8
    out.hostsim_epilogue.restype = C.c_int
    return out


@pytest.mark.parametrize("max_steps,split", [(5, False), (5, True)])
@pytest.mark.parametrize("name,kwargs", SCENARIOS)
def test_epilogue_takes_the_count_it_is_handed(name, kwargs, max_steps, split):
    B = 48
    env = _env(name, kwargs, max_steps, split, n_envs=B, steps=20)
    prog, instrs, limit, merged, _, slots, _ = _programs(env)
    lib = _compile(P.describe_world(env.world), merged, f"{name}_{max_steps}_{int(split)}")
    counts = (np.arange(B) % 9).astype(np.float32)
    counts[-1] = 2.0 ** 24  # (max_steps = 5: far past it)
    slab = env.world.slab
    state = {k: np.ascontiguousarray(getattr(slab, k).numpy().astype(np.float32))
             for k in ("pos", "vel", "rot", "ang_vel", "force", "torque")}
    n_slots = len(prog.buffers)
    inputs = [prog.resolve(b).numpy().copy() if prog.resolve(b).dtype != torch.bool else np.zeros(B, np.uint8)
              for b in prog.buffers]
    counter = slots[limit.count_slot]

    def run(G, handed):
        arr = {k: v.copy() for k, v in state.items()}
        bufs = [x.copy() for x in inputs] + [np.zeros(B, np.uint8) for _ in slots]
        # the counter's buffer: the counts themselves for the load, else poison
        bufs[counter] = counts.copy() if handed is None else np.full(B, np.nan, np.float32)
        ptrs = (C.c_void_p * 32)()
        for slot, b in enumerate(bufs):
            ptrs[slot] = b.ctypes.data
        assert lib.hostsim_epilogue(G, B, *(arr[k].ctypes.data for k in ("pos", "vel", "rot", "ang_vel", "force", "torque")),
                                    None if handed is None else handed.ctypes.data, ptrs) == 0
        return bufs

    loaded = run(1, None)
    for G in (1, 2):
        got = run(G, counts)
        for slot in range(n_slots + len(slots)):
            if slot != counter:
                assert np.array_equal(got[slot].view(np.uint8), loaded[slot].view(np.uint8)), f"G = {G}: buffer {slot}"
    # against the oracle: the scenario's program, then the limit program reading the counter
    env.steps.copy_(torch.from_numpy(counts))
    with use_oracle():
        prog.run()
        env._limit_input = prog.out_done.tensor
        limit.run()
    out = limit.out.tensor.numpy()
    assert np.array_equal(loaded[slots[limit.out._slot]].astype(bool), out)
    assert out.any() and not out.all()
    want = _torch_statements(env, prog.out_done.tensor)
    assert np.array_equal(out, want.numpy())
    for slot, b in enumerate(prog.buffers):
        t = prog.resolve(b)
        if t.dtype == torch.bool:
            assert np.array_equal(loaded[slot].astype(bool), t.numpy()), f"bool buffer {slot}"
        else:
            assert np.allclose(loaded[slot], t.numpy(), rtol=1e-4, atol=2e-4), f"buffer {slot}"
