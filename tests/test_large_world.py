"""Worlds past the thread-per-env step's shared-memory limit, without a GPU.

* The CPU oracle equals the reference's recorded roll-outs of the large crafted worlds
  (``tests/crafted_large.py``: 160, 520 and 1024 entities) bit for bit, as ``test_oracle_vs_reference.py``
  checks for the other fixtures.
* hostsim: the block-per-env kernel's phases (``csrc/generic_step.cuh``, the block's threads run one after the
  other between barriers, shared memory poisoned with NaN) against the item-order walk of the thread-per-env
  kernel, built from the same header by the same compiler: the same bits on every golden world, on the
  per-env-parameter world and on the three large worlds, with and without broad-phase masks; within the
  libm tolerance of the reference's results.  A descending incidence list and a dropped side of a work item
  are both caught.
* Mapping selection on a ``cpu`` device: every golden world keeps its ``auto`` mapping, the 160-entity world
  gets the block-per-env kernel, and a world past 1024 entities is refused when its plan is uploaded.
"""
import ctypes as C
import os
import subprocess
import types

import numpy as np
import pytest
import torch

import golden_pack
from golden_util import GOLDEN_DIR, STATE_KEYS, golden_names, load, teacher_forced_steps
from oracle import world_step as WS
from vectorizedmultiagentsimulator_b200 import _native
from vectorizedmultiagentsimulator_b200.simulator import plan as P

HERE = os.path.dirname(os.path.abspath(__file__))
SIM_DIR = os.path.join(HERE, "hostsim")
SIM_LIB = os.path.join(SIM_DIR, "_block_step.so")
LARGE = ("large_160-0", "large_520-1", "large_1024-2")
STATE = ("pos", "vel", "rot", "ang_vel")
COLS = {"mass": P.EP_MASS, "linear_friction": P.EP_LIN_FRIC, "angular_friction": P.EP_ANG_FRIC}


def load_large(case):
    rec = golden_pack.load(os.path.join(GOLDEN_DIR, "reference", "teacher_forced", case + ".npz"))
    desc = P.WorldDescription.from_json(rec["desc"])
    return rec, desc, P.build_tables(desc)


def _same(got, want, rec):
    """Bit for bit on the vector ISA the reference ran on; elsewhere within the 2e-6 of test_oracle_golden.py."""
    if rec["cpu_capability"] == torch.backends.cpu.get_cpu_capability():
        return torch.equal(got, want)
    return got.shape == want.shape and float((got - want).abs().max()) <= 2e-6


@pytest.mark.parametrize("case", LARGE)
def test_oracle_equals_reference_on_large_worlds(case):
    rec, desc, tables = load_large(case)
    assert desc.n_entities == int(case.split("_")[1].split("-")[0])
    assert tables.n_masked > 32 * 32 and desc.n_joints == 4  # two joints, two constraints each
    for t, state_in, fixed_rot, want in teacher_forced_steps(rec):
        state = {k: state_in[k] for k in STATE_KEYS}
        WS.world_step(tables, state, fixed_rot=fixed_rot)
        for k in STATE:
            assert _same(state[k], want[k], rec), f"{case} step {t}: {k} max |diff| {float((state[k] - want[k]).abs().max())}"


def ulp_sensitivity(tables, state_in, fixed_rot, trials=3):
    """max |oracle(x) - oracle(x perturbed by +-1 ulp)| per field: the joint envelope of DESIGN.md section 6.
    The large worlds are joint worlds, and their packed contacts amplify a last-bit difference too."""
    base = {k: state_in[k].clone() for k in STATE_KEYS}
    WS.world_step(tables, base, fixed_rot=fixed_rot)
    gen = torch.Generator().manual_seed(0)
    worst = {k: 0.0 for k in STATE_KEYS}
    for _ in range(trials):
        pert = {k: state_in[k].clone() for k in STATE_KEYS}
        for k in ("pos", "rot"):
            sign = torch.randint(0, 3, pert[k].shape, generator=gen).float() - 1.0
            pert[k] = pert[k] * (1.0 + sign * 2.0**-23)
        WS.world_step(tables, pert, fixed_rot=fixed_rot)
        for k in STATE_KEYS:
            worst[k] = max(worst[k], float((pert[k] - base[k]).abs().max()))
    return worst


# ---- hostsim ---------------------------------------------------------------------------------
def _build():
    sources = [os.path.join(SIM_DIR, "block_step.cpp"), os.path.join(SIM_DIR, "shim", "cuda_runtime.h")] + _native.HEADERS
    if os.path.exists(SIM_LIB) and all(os.path.getmtime(f) <= os.path.getmtime(SIM_LIB) for f in sources):
        return
    subprocess.run(
        ["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-DVMAS_HOSTSIM",
         "-I", os.path.join(SIM_DIR, "shim"), "-I", _native.CSRC, "-I", _native.INCLUDE,
         os.path.join(SIM_DIR, "block_step.cpp"), "-o", SIM_LIB],
        check=True,
    )


@pytest.fixture(scope="module")
def sim():
    _build()
    lib = C.CDLL(SIM_LIB)
    lib.hostsim_generic_step.argtypes = [C.c_int, C.c_void_p, C.c_void_p] + [C.c_void_p] * 8 + [C.c_int] * 3
    lib.hostsim_generic_step.restype = C.c_int
    return lib


def _host_tables(tables, B, fixed_rot=None, ent_gravity=None, ent_params=None):
    """The plan tables as the backend uploads them, in host memory (DeviceTables on the cpu device)."""
    dt = _native.DeviceTables(tables, None, torch.device("cpu"), mapping="thread_per_env")
    dt.cfg.batch_dim = B
    for k, v in (fixed_rot or {}).items():
        dt.joint_rot[:, k] = v.reshape(-1)
    for e, g in (ent_gravity or {}).items():
        dt.ent_gravity[:, e] = g
    for e, values in (ent_params or {}).items():
        for attr, v in values.items():
            if attr in COLS:
                dt.ent_params[:, e, COLS[attr]] = v.reshape(-1)
    return dt


def _with_incidence(dt, inc_off, inc):
    """``dt`` with its incidence lists replaced (host arrays kept alive on the object)."""
    dt.mut = (np.ascontiguousarray(inc_off, np.int32), np.ascontiguousarray(inc, np.int32))
    dt.tb.inc_off = dt.mut[0].ctypes.data
    dt.tb.inc = dt.mut[1].ctypes.data
    return dt


def _run(lib, variant, dt, state, mask=None, first=0, n=None):
    arr = {k: np.ascontiguousarray(state[k].numpy().astype(np.float32)).copy() for k in STATE_KEYS}
    B = arr["pos"].shape[0]
    cfg = dt.cfg
    cfg.batch_dim = B
    params = None if dt.ent_params is None else dt.ent_params.data_ptr()
    m = None if mask is None else np.asarray(mask, np.uint32)
    rc = lib.hostsim_generic_step(
        variant, C.byref(cfg), C.byref(dt.tb), *(arr[k].ctypes.data for k in STATE_KEYS), params,
        None if m is None else m.ctypes.data, int(m is not None), first, cfg.substeps if n is None else n,
    )
    assert rc == 0
    return arr


def _masked_step(lib, dt, tables, state):
    """One World.step of the block formulation as the backend runs it: per substep the batch-wide
    broad-phase mask of the current positions (the oracle's), then one substep."""
    cur = {k: v.clone() for k, v in state.items() if k in STATE_KEYS}
    items = [int(k) for k in tables.masked_items[: tables.n_masked]]
    for sub in range(tables.desc.substeps):
        on = WS.broad_phase_active_many(tables, items, cur["pos"])
        words = np.zeros((tables.n_masked + 31) // 32, np.uint32)
        for j, active in enumerate(on):
            words[j >> 5] |= np.uint32(active) << np.uint32(j & 31)
        out = _run(lib, 1, dt, cur, words, sub, 1)
        cur = {k: torch.from_numpy(v) for k, v in out.items()}
    return {k: v.numpy() for k, v in cur.items()}


def _cases():
    """(name, tables, [(t, state_in, fixed_rot, ent_gravity, ent_params, want)]) of every world checked."""
    for name in golden_names():
        fix, desc, tables = load(name)
        steps = [(t, s, fr, s.get("ent_gravity"), None, w) for t, s, fr, w in teacher_forced_steps(fix) if t % 4 == 0]
        yield name, tables, steps
    params = golden_pack.load(os.path.join(GOLDEN_DIR, "reference", "teacher_forced", "crafted_randomised-0.npz"))
    tables = P.build_tables(P.WorldDescription.from_json(params["desc"]))
    steps = [(t, s, fr, e["ent_gravity"], e["ent_params"], w)
             for (t, s, fr, w), e in zip(teacher_forced_steps(params), params["steps"]) if t % 3 == 0]
    yield "crafted_randomised", tables, steps
    for case in LARGE:
        rec, _, tables = load_large(case)
        yield case, tables, [(t, s, fr, None, None, w) for t, s, fr, w in teacher_forced_steps(rec)]


CASES = list(_cases())


@pytest.mark.parametrize("i", range(len(CASES)), ids=[c[0] for c in CASES])
def test_block_phases_equal_item_order_walk_bitwise(sim, i):
    name, tables, steps = CASES[i]
    words = (tables.n_masked + 31) // 32
    substeps = tables.desc.substeps
    rng = np.random.default_rng(i)
    for t, state_in, fixed_rot, ent_gravity, ent_params, want in steps:
        dt = _host_tables(tables, state_in["pos"].shape[0], fixed_rot, ent_gravity, ent_params)
        masks = [None] + ([rng.integers(0, 2**32, words, dtype=np.uint64).astype(np.uint32) for _ in range(2)] if words else [])
        for mask in masks:
            # with a mask, one substep per launch, as the backend launches them
            first, n = (0, substeps) if mask is None else (min(1, substeps - 1), 1)
            a = _run(sim, 0, dt, state_in, mask, first, n)
            b = _run(sim, 1, dt, state_in, mask, first, n)
            for k in STATE_KEYS:
                assert np.array_equal(a[k], b[k]), f"{name} step {t} field {k} (mask {mask is not None})"
            assert all(np.isfinite(b[k]).all() for k in STATE_KEYS), f"{name} step {t}: a poisoned value was read"
        if name in LARGE:  # libm is not CUDA's: against the reference within the GPU tests' tolerance
            got = _masked_step(sim, dt, tables, state_in)
            sens = ulp_sensitivity(tables, state_in, fixed_rot)
            for k in STATE:
                w = want[k].numpy().reshape(got[k].shape)
                err = np.abs(got[k] - w)
                atol = 1e-5 + 4.0 * sens[k]
                assert np.all(err <= atol + 1e-4 * np.abs(w)), f"{name} step {t} {k}: max |err| {err.max()} (atol {atol:.2e})"


def _mutated(tables, how):
    """Incidence lists of ``tables`` with each entity's list reversed, or with item 0's second side dropped."""
    off, inc = tables.inc_off.astype(np.int64), tables.inc.copy()
    if how == "descending":
        for e in range(len(off) - 1):
            inc[off[e]:off[e + 1]] = inc[off[e]:off[e + 1]][::-1].copy()
        return off, inc
    drop = int(np.nonzero(inc[: off[-1]] == 1)[0][0])  # item 0, side b
    owner = int(np.searchsorted(off, drop, side="right")) - 1
    off = off.copy()
    off[owner + 1:] -= 1
    return off, np.delete(inc[: tables.inc_off[-1]], drop)


@pytest.mark.parametrize("how", ["descending", "drop_side"])
def test_block_phases_catch_a_wrong_incidence_list(sim, how):
    rec, desc, tables = load_large("large_160-0")
    _, state_in, fixed_rot, _ = next(teacher_forced_steps(rec))
    B = state_in["pos"].shape[0]
    want = _run(sim, 0, _host_tables(tables, B, fixed_rot), state_in)
    same = _run(sim, 1, _host_tables(tables, B, fixed_rot), state_in)
    assert all(np.array_equal(want[k], same[k]) for k in STATE_KEYS)
    bad = _run(sim, 1, _with_incidence(_host_tables(tables, B, fixed_rot), *_mutated(tables, how)), state_in)
    assert not all(np.array_equal(want[k], bad[k]) for k in STATE_KEYS), how


# ---- mapping selection -------------------------------------------------------------------------
def test_auto_mapping_keeps_every_golden_world_and_picks_blocks_past_the_tpe_limit():
    cpu = torch.device("cpu")
    lib = _native.load()
    from vectorizedmultiagentsimulator_b200 import codegen

    for name in golden_names():
        _, desc, tables = load(name)
        dt = _native.DeviceTables(tables, None, cpu, mapping="auto")
        specialised = lib.vmas_b200_find_specialization(codegen.world_hash(desc)) >= 0
        assert dt.mapping == (_native.DEFAULT_SPEC_MAPPING if specialised else "thread_per_env"), name
        assert _native.tpe_fits(tables, cpu), name
    _, desc, tables = load_large("large_160-0")
    assert not _native.tpe_fits(tables, cpu)
    dt = _native.DeviceTables(tables, None, cpu, mapping="auto")
    assert dt.mapping == "block_per_env" and dt.tb.group == _native.GROUP_BLOCK and dt.tb.specialization == -1
    # explicit: the block-per-env kernel on a small world
    _, _, small = load("balance")
    dt = _native.DeviceTables(small, None, cpu, mapping="block_per_env")
    assert dt.mapping == "block_per_env" and dt.tb.group == _native.GROUP_BLOCK and dt.tb.specialization == -1


def test_tpe_limit_is_the_shared_memory_of_32_envs():
    fake = lambda E, masked: types.SimpleNamespace(desc=types.SimpleNamespace(n_entities=E), n_masked=masked)  # noqa: E731
    cpu = torch.device("cpu")
    assert _native.shared_optin_bytes(cpu) == 232448
    assert _native.tpe_fits(fake(139, 0), cpu) and not _native.tpe_fits(fake(140, 0), cpu)
    # 139 entities leave 1 152 bytes: 288 mask words
    assert _native.tpe_fits(fake(139, 288 * 32), cpu) and not _native.tpe_fits(fake(139, 288 * 32 + 1), cpu)


def test_world_past_1024_entities_is_refused_at_plan_upload():
    _, desc, _ = load_large("large_1024-2")
    desc.entities.append(dict(desc.entities[-1]))
    assert desc.n_entities == 1025
    tables = P.build_tables(desc)
    for mapping in ("auto", "thread_per_env", "block_per_env"):
        with pytest.raises(NotImplementedError, match="1024"):
            _native.DeviceTables(tables, None, torch.device("cpu"), mapping=mapping)
