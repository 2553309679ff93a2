"""The C-ABI library builds, loads and exports every symbol include/vmas_b200.h declares."""
import ctypes
import os
import re

from vectorizedmultiagentsimulator_b200 import _native

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    text = open(os.path.join(ROOT, "include", "vmas_b200.h")).read()
    return sorted(set(re.findall(r"\b(vmas_b200_\w+)\s*\(", text)))


def test_header_symbols_are_exported():
    _native.build()
    lib = ctypes.CDLL(_native.LIB_PATH)
    symbols = declared_symbols()
    assert len(symbols) >= 8
    for name in symbols:
        assert hasattr(lib, name), f"{name} declared in vmas_b200.h but not exported"
    assert sorted(_native.EXPORTS) == symbols


def test_abi_version_and_struct_sizes():
    lib = _native.load()
    assert lib.vmas_b200_abi_version() == 2
    # 10 int32 + 9 float
    assert ctypes.sizeof(_native.WorldConfig) == 19 * 4
    assert ctypes.sizeof(_native.PlanTablesC) == 10 * 8 + 4 * 4 + 2 * 8  # + env_order, env_signature (ABI 2)
    assert ctypes.sizeof(_native.StateC) == 6 * 8


def test_argument_validation_without_gpu():
    """Error paths that return before any CUDA call."""
    lib = _native.load()
    assert lib.vmas_b200_world_step(None, None, None, None, 1, None) < 0
    assert b"null" in lib.vmas_b200_last_error()


def test_reset_entry_points_validate_their_arguments_without_gpu():
    """vmas_b200_reset_state / vmas_b200_spawn_entities reject bad input before any CUDA call."""
    lib = _native.load()
    cfg = _native.WorldConfig()
    cfg.batch_dim, cfg.n_entities, cfg.n_agents = 16, 4, 2
    st = _native.StateC()
    st.pos = st.vel = st.rot = st.ang_vel = st.force = st.torque = 0x1000  # never dereferenced on the host

    def err():
        return lib.vmas_b200_last_error().decode()

    assert lib.vmas_b200_reset_state(None, None, -1, None, None, None) < 0 and "null" in err()
    assert lib.vmas_b200_reset_state(ctypes.byref(cfg), ctypes.byref(st), 16, None, None, None) < 0
    assert "env_index" in err()

    def spawn(**kw):
        sp = _native.SpawnC()
        sp.n_spawn, sp.max_tries, sp.env_index = 2, 100, -1
        sp.entity[0], sp.entity[1] = 0, 1
        sp.x_lo, sp.x_hi, sp.y_lo, sp.y_hi, sp.min_dist = -1, 1, -1, 1, 0.1
        for k, v in kw.items():
            setattr(sp, k, v)
        return lib.vmas_b200_spawn_entities(ctypes.byref(cfg), ctypes.byref(st), ctypes.byref(sp), None)

    assert spawn(n_spawn=0) < 0 and "n_spawn" in err()
    assert spawn(n_spawn=_native.MAX_SPAWN + 1) < 0 and "n_spawn" in err()
    assert spawn(max_tries=0) < 0 and "max_tries" in err()
    assert spawn(env_index=16) < 0 and "env_index" in err()
    assert spawn(x_lo=2.0) < 0 and "bounds" in err()
    assert spawn(n_occupied=3) < 0 and "occupied" in err()
    sp = _native.SpawnC()
    sp.n_spawn, sp.max_tries, sp.env_index = 1, 10, -1
    sp.entity[0] = 9
    sp.x_hi = sp.y_hi = 1.0
    assert lib.vmas_b200_spawn_entities(ctypes.byref(cfg), ctypes.byref(st), ctypes.byref(sp), None) < 0
    assert "out of range" in err()
    sp.entity[0] = -1  # position only, but no `out` buffer either
    assert lib.vmas_b200_spawn_entities(ctypes.byref(cfg), ctypes.byref(st), ctypes.byref(sp), None) < 0
    assert "nothing to write" in err()


def test_device_tables_build_for_every_mapping_on_cpu():
    """The host-side table upload of each thread mapping (incl. the warp-tile one) — what
    runs before the first launch — without a GPU."""
    import sys

    import pytest
    import torch

    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from golden_util import load

    cpu = torch.device("cpu")
    for name, specialised in (("balance", True), ("flocking", True), ("pollock", False)):
        _, desc, tables = load(name)
        auto = _native.DeviceTables(tables, None, cpu, mapping="auto")
        assert auto.mapping == ((_native.DEFAULT_SPEC_MAPPING if specialised else "thread_per_env"))
        for mapping in ("thread_per_env", "lanes_per_env"):
            dt = _native.DeviceTables(tables, None, cpu, mapping=mapping)
            assert dt.mapping == mapping and dt.tb.specialization == -1 and dt.tb.group >= 1
        for mapping, group in (("specialized", 1), ("tile", _native.GROUP_TILE)):
            if specialised:
                dt = _native.DeviceTables(tables, None, cpu, mapping=mapping)
                assert dt.mapping == mapping and dt.tb.group == group and dt.tb.specialization >= 0
                assert dt.tb.specialization == auto.tb.specialization
            else:
                with pytest.raises(RuntimeError):
                    _native.DeviceTables(tables, None, cpu, mapping=mapping)
        with pytest.raises(ValueError, match="auto, specialized, tile, thread_per_env, lanes_per_env, block_per_env"):
            _native.DeviceTables(tables, None, cpu, mapping="warp")


def test_ctypes_structs_have_the_layout_of_the_c_header(tmp_path):
    """Every ctypes mirror of a C-ABI struct: same field names, offsets and total size as ``include/vmas_b200.h``
    gives them (checked by compiling a few ``offsetof`` lines with gcc) — a field inserted on one side only
    would otherwise shift pointers silently."""
    import subprocess

    pairs = [
        (_native.WorldConfig, "VmasWorldConfig"), (_native.PlanTablesC, "VmasPlanTables"), (_native.StateC, "VmasState"),
        (_native.AgentActionsC, "VmasAgentActions"), (_native.ProgInstrC, "VmasProgInstr"),
        (_native.StepProgramC, "VmasStepProgram"), (_native.CopySegmentC, "VmasCopySegment"),
        (_native.EnvStepC, "VmasEnvStep"),
    ]
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "vmas_b200.h"', "int main(void) {"]
    for cls, cname in pairs:
        lines.append(f'  printf("%zu\\n", sizeof({cname}));')
        for field, *_ in cls._fields_:
            lines.append(f'  printf("%zu\\n", offsetof({cname}, {field}));')
    lines += ["  return 0;", "}"]
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text("\n".join(lines))
    subprocess.run(["gcc", "-I", _native.INCLUDE, str(src), "-o", str(exe)], check=True)
    got = iter(int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split())
    for cls, cname in pairs:
        assert ctypes.sizeof(cls) == next(got), f"sizeof({cname})"
        for field, *_ in cls._fields_:
            assert getattr(cls, field).offset == next(got), f"{cname}.{field}"
