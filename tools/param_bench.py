"""ms per ``World.step`` of the per-env-parameter world (tests/crafted_params.py) on the generic and on the run-time
specialised kernel, with the card's name and power limit.

    python tools/param_bench.py [--envs 32768] [--steps 200]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = torch.cuda.get_device_name(0) + ", power limit unknown"
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=32768)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    import crafted_params
    import vectorizedmultiagentsimulator_b200 as b200
    from vectorizedmultiagentsimulator_b200 import _native

    env = b200.make_env(crafted_params.make_scenario("vectorizedmultiagentsimulator_b200"), num_envs=args.envs,
                        device="cuda:0", seed=0)
    world = env.world
    backend = world._get_backend()
    backend.wait_for_jit()
    result = dict(card=card(), envs=args.envs, steps=args.steps)
    for mapping in ("thread_per_env", "specialized"):
        backend._dev_tables = _native.DeviceTables(backend.tables, world, backend.device, mapping=mapping)
        assert backend._dev_tables.mapping == mapping
        for _ in range(args.warmup):
            world.step()
        begin, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        begin.record()
        for _ in range(args.steps):
            world.step()
        end.record()
        torch.cuda.synchronize()
        result[f"ms_per_step_{mapping}"] = begin.elapsed_time(end) / args.steps
    print(json.dumps(result))


if __name__ == "__main__":
    main()
