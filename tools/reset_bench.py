"""Cost of resetting finished envs (SURVEY §8(f)-4), on one GPU.

    python tools/reset_bench.py

For each scenario: wall-clock (host + device, synchronised) of
  * ``reset_at(mask)`` with 25 % of the envs flagged — device-side reset (this library's kernels);
  * the same call with ``VMAS_B200_DEVICE_RESET=0`` — the reference's formulation in torch ops on
    the GPU (python ``while`` loop with a host sync per attempt, masked writes);
  * one ``reset_at(i)`` (what the reference API offers: a training loop calls it once per finished
    env), in both modes; the cost of resetting N finished envs that way is N times this.
One JSON line per (scenario, mode).  Not a bench.py value: wall-clock around a synchronised region.
"""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch

import vectorizedmultiagentsimulator_b200 as b200
from vectorizedmultiagentsimulator_b200.simulator.core import World

CONFIGS = [
    ("balance", 32768, dict(n_agents=4)),
    ("transport", 16384, dict(n_agents=4)),
    ("navigation", 8192, dict(n_agents=8)),
    ("flocking", 32768, dict(n_agents=5)),
]


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps


def main():
    for name, B, kwargs in CONFIGS:
        for device_reset in (True, False):
            World.device_reset_enabled = device_reset
            env = b200.make_env(name, num_envs=B, device="cuda", seed=0, **kwargs)
            gen = torch.Generator().manual_seed(0)
            mask = (torch.rand(B, generator=gen) < 0.25).cuda()
            backend = env.world._get_backend()
            l0 = backend.launches
            t_mask = timed(lambda: env.reset_at(mask, return_observations=False), 10)
            launches = (backend.launches - l0) // 11
            t_one = timed(lambda: env.reset_at(7, return_observations=False), 20)
            t_all = timed(lambda: env.reset(return_observations=False), 10)
            print(json.dumps({
                "scenario": name, "num_envs": B, "kwargs": kwargs,
                "mode": "device_reset" if device_reset else "torch_ops",
                "reset_at_mask_25pct_ms": round(t_mask * 1e3, 3),
                "envs_reset_per_call": int(mask.sum()),
                "library_launches_per_masked_reset": launches,
                "reset_at_one_env_ms": round(t_one * 1e3, 3),
                "reset_all_ms": round(t_all * 1e3, 3),
                "spawn_failures": env.world.spawn_failures(),
            }), flush=True)
            del env
    World.device_reset_enabled = True


main()
