"""Run-time specialisation (vectorizedmultiagentsimulator_b200/jit.py) without a GPU: the world's tables are
emitted, nvcc cross-compiles the object for sm_90a, its launch functions are registered with the
main library and the plan upload then selects the specialised mapping.  (Launching it is
tests/test_cabi_gpu.py::test_runtime_specialisation_agrees_bitwise, on the GPU.)"""
import pytest
import torch

from golden_util import load
from vectorizedmultiagentsimulator_b200 import _native, codegen, jit


@pytest.mark.parametrize("name", ["give_way", "crafted_clamps"])
def test_world_without_a_preset_gets_a_specialisation(name, tmp_path, monkeypatch):
    if not jit.available():
        pytest.skip("no nvcc / JIT switched off")
    monkeypatch.setattr(jit, "CACHE_DIR", str(tmp_path))
    _, desc, tables = load(name)
    lib = _native.load()
    h = codegen.world_hash(desc)
    if lib.vmas_b200_find_specialization(h) >= 0:
        pytest.skip("already registered by an earlier test of this process")
    cpu = torch.device("cpu")
    assert _native.DeviceTables(tables, None, cpu, mapping="auto").mapping == "thread_per_env"
    job = jit.request(desc)
    assert job is not None
    assert job.done.wait(timeout=300), "nvcc did not finish"
    assert job.error is None, job.error
    assert job.index >= lib.vmas_b200_num_specializations() - 256 and lib.vmas_b200_find_specialization(h) == job.index
    dt = _native.DeviceTables(tables, None, cpu, mapping="auto")
    assert dt.mapping == _native.DEFAULT_SPEC_MAPPING or dt.mapping == "specialized"
    assert dt.tb.specialization == job.index
    assert jit.request(desc) is job  # one compilation per world and process
    assert list(tmp_path.glob("*.so")), "the object is cached on disk"


def test_worlds_that_cannot_be_specialised_are_left_alone():
    _, desc, _ = load("pollock")  # 990 work items: over the unrolling budget
    assert jit.request(desc) is None
