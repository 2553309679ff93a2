"""ms per ``World.step`` of large worlds (tests/crafted_large.py) on the block-per-env kernel, the thread-per-env
kernel where an env's state fits its shared memory, and the CPU oracle's torch op chain run on the GPU, with
the card's name and power limit.

    python tools/large_world_bench.py [--sizes 70,139,160,256,512,1024] [--envs 256,4096,32768] [--out f.json]

Per (entities, envs): eager ``World.step`` and a CUDA graph of it replayed, timed with CUDA events after a
warm-up over a window of at least ``--window`` seconds; the two kernels alternate in the same process.  Also
the plan-build time (``describe_world`` + ``build_tables``) per world size.  One JSON line per measurement.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out or torch.cuda.get_device_name(0) + ", power limit unknown"


def timed(fn, window, warmup=3):
    """Mean ms per call of ``fn`` over a window of >= ``window`` seconds (CUDA events, after ``warmup`` calls)."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    begin, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    begin.record()
    fn()
    end.record()
    torch.cuda.synchronize()
    n = int(min(500, max(5, window * 1e3 / max(begin.elapsed_time(end), 1e-3))))
    begin.record()
    for _ in range(n):
        fn()
    end.record()
    torch.cuda.synchronize()
    return begin.elapsed_time(end) / n, n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="70,139,160,256,512,1024")
    ap.add_argument("--envs", default="256,4096,32768")
    ap.add_argument("--window", type=float, default=0.5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import crafted_large
    import vectorizedmultiagentsimulator_b200 as b200
    from oracle import world_step as WS
    from vectorizedmultiagentsimulator_b200 import _native
    from vectorizedmultiagentsimulator_b200.simulator import plan as P

    lines = []

    def emit(rec):
        print(json.dumps(rec), flush=True)
        lines.append(rec)

    emit(dict(card=card(), torch=torch.__version__))
    for E in (int(s) for s in args.sizes.split(",")):
        for B in (int(s) for s in args.envs.split(",")):
            rec = dict(entities=E, envs=B)
            try:
                env = b200.make_env(crafted_large.make_scenario("vectorizedmultiagentsimulator_b200", f"large_{E}"),
                                    num_envs=B, device="cuda:0", seed=0)
            except torch.cuda.OutOfMemoryError:
                emit(dict(rec, error="out of memory"))
                continue
            world = env.world
            t0 = time.perf_counter()
            desc = P.describe_world(world)
            t1 = time.perf_counter()
            tables = P.build_tables(desc)
            t2 = time.perf_counter()
            rec.update(items=len(desc.items), describe_world_s=round(t1 - t0, 4), build_tables_s=round(t2 - t1, 4))
            backend = world._get_backend()
            world.step()
            rec["auto_mapping"] = backend._dev_tables.mapping
            saved = world.slab.state_dict()
            mappings = ["block_per_env"] + (["thread_per_env"] if _native.tpe_fits(tables, backend.device) else [])
            for rnd in range(2):  # the kernels alternate: two rounds each
                for mapping in mappings:
                    backend._dev_tables = _native.DeviceTables(backend.tables, world, backend.device, mapping=mapping)
                    world.slab.load_state_dict(saved)
                    ms, n = timed(world.step, args.window)
                    rec.setdefault(f"eager_ms_{mapping}", []).append(round(ms, 5))
                    world.slab.load_state_dict(saved)
                    try:
                        g = torch.cuda.CUDAGraph()
                        s = torch.cuda.Stream()
                        s.wait_stream(torch.cuda.current_stream())
                        with torch.cuda.stream(s):
                            world.step()
                            torch.cuda.synchronize()
                            with torch.cuda.graph(g):
                                world.step()
                        torch.cuda.current_stream().wait_stream(s)
                        ms, n = timed(g.replay, args.window)
                        rec.setdefault(f"graph_ms_{mapping}", []).append(round(ms, 5))
                        rec[f"steps_timed_{mapping}"] = n
                        del g
                    except RuntimeError as exc:  # reported, not hidden
                        rec[f"graph_ms_{mapping}"] = f"capture failed: {str(exc)[:160]}"
            # the reference arm: the oracle's torch op chain on the same GPU, on the same state
            state = {k: v.clone() for k, v in saved.items() if k in ("pos", "vel", "rot", "ang_vel", "force", "torque")}

            def oracle_step():
                with torch.device(backend.device):  # the oracle's constant tensors on the GPU too
                    WS.world_step(tables, state)

            try:
                ms, n = timed(oracle_step, args.window, warmup=1)
                rec["oracle_torch_gpu_ms"] = round(ms, 4)
            except Exception as exc:  # noqa: BLE001 - reported, not hidden
                rec["oracle_torch_gpu_ms"] = f"failed: {type(exc).__name__}: {str(exc)[:120]}"
            emit(rec)
            del env, world, backend, saved, state
            torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(lines, fh, indent=1)


if __name__ == "__main__":
    main()
