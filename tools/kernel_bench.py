"""Times the substep kernel alone (both thread mappings) on a tiled golden state.

    python tools/kernel_bench.py [scenario ...] [batch size ...]       # on a GPU
    KB_MAPPINGS=specialized VMAS_B200_LIB=tools/variants/lib_x.so python tools/kernel_bench.py balance
"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
from golden_util import STATE_KEYS, load, teacher_forced_steps
from vectorizedmultiagentsimulator_b200 import _native
from vectorizedmultiagentsimulator_b200.simulator import plan as P
from test_cabi_gpu import _Slab

lib = _native.load()
if os.environ.get("VMAS_B200_L2_FETCH"):
    print("# L2 fetch granularity:", lib.vmas_b200_set_l2_fetch_granularity(int(os.environ["VMAS_B200_L2_FETCH"])))
dev = torch.device("cuda:0")
peak = 3350.0  # GB/s: NVIDIA H100 SXM data sheet (HBM3)
flush = torch.empty(512 << 20, dtype=torch.uint8, device=dev)
names = [a for a in sys.argv[1:] if not a.isdigit()] or ["balance", "transport", "navigation", "flocking", "pollock"]
sizes = [int(a) for a in sys.argv[1:] if a.isdigit()] or [32768, 1 << 20]
for name in names:
    fix, desc, tables = load(name)
    steps = list(teacher_forced_steps(fix))
    _, state_in, fixed_rot, _ = steps[min(5, len(steps) - 1)]
    bpe = P.algorithmic_bytes_per_env_substep(desc)
    for B in sizes:
        reps = max(1, B // desc.batch_dim)
        big = {k: v.repeat(reps, *([1] * (v.dim() - 1))) for k, v in state_in.items()}
        Bn = big["pos"].shape[0]
        for mapping in os.environ.get("KB_MAPPINGS", "specialized,thread_per_env,lanes_per_env").split(","):
            # "specialized_ordered": the thread-per-env kernel with its envs scheduled by contact signature
            ordered = mapping.endswith("_ordered")
            _native.ENV_REORDER_EVERY = 8 if ordered else 0
            old = desc.batch_dim
            desc.batch_dim = Bn
            try:
                dt = _native.DeviceTables(tables, None, dev, mapping=mapping.replace("_ordered", ""))
            except RuntimeError:
                desc.batch_dim = old
                continue
            desc.batch_dim = old
            slab = _Slab(big, dev)
            saved = {k: slab.t[k].clone() for k in STATE_KEYS}
            if ordered:
                if dt.env_order is None:
                    continue
                _native.world_step(lib, dt, slab)  # records the signatures of this state
                _native.build_env_order(lib, dt)
                torch.cuda.synchronize()
                order = dt.env_order.long()
                assert torch.equal(torch.sort(order).values, torch.arange(Bn, device=dev)), "order is not a permutation"
            times = []
            for it in range(12):
                for k in STATE_KEYS:
                    slab.t[k].copy_(saved[k])
                flush.zero_()
                ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
                _native.world_step(lib, dt, slab, events=ev)
                torch.cuda.synchronize()
                times.append(ev[0].elapsed_time(ev[1]) * 1e3)
            times = sorted(times[2:])
            us = times[len(times) // 2]
            launches_per_step = desc.substeps if tables.n_masked else 1
            gbs = bpe * Bn * launches_per_step / us / 1e3
            print(f"{name:12s} B={Bn:8d} {mapping:15s} {us:9.1f} us/step  S={desc.substeps} "
                  f"bytes/env/substep={bpe}  {gbs:8.1f} GB/s  frac={gbs/peak:.3f}")
