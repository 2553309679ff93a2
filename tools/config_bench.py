"""env-steps/s of Environment.step (CUDA-graph mode) on the BASELINE.json configs C2-C5 at 1 GPU.

    python tools/config_bench.py

One JSON line per config: CUDA events around each step, 512 MiB L2 flush between steps (outside
the events), actions resident on the device.  C5 is run at the per-GPU share of an 8-GPU job
(32768 envs) and at the full 262144 envs on one GPU.
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch

import vectorizedmultiagentsimulator_b200 as b200

CONFIGS = [
    ("C2 balance", "balance", 32768, dict(n_agents=4)),
    ("C3 transport (stock)", "transport", 16384, dict(n_agents=4)),
    ("C3 transport (+2 lines, 3 substeps)", "transport", 16384, dict(n_agents=4, n_lines=2, substeps=3)),
    ("C4 navigation", "navigation", 8192, dict(n_agents=8)),
    ("C5 flocking (1/8 share)", "flocking", 32768, dict(n_agents=5)),
    ("C5 flocking (whole job on 1 GPU)", "flocking", 262144, dict(n_agents=5)),
]


def main():
    steps, warmup = 100, 5
    flush = torch.empty(512 << 20, dtype=torch.uint8, device="cuda")
    for label, name, B, kwargs in CONFIGS:
        for graph in (True, False):
            env = b200.make_env(name, num_envs=B, device="cuda", seed=0, cuda_graph=graph, **kwargs)
            env.reset()
            gen = torch.Generator().manual_seed(1)
            acts = [
                [(torch.rand(B, a.action_size, generator=gen) * 2 - 1).cuda() for a in env.agents] for _ in range(16)
            ]
            for i in range(warmup):
                env.step(acts[i % 16])
            torch.cuda.synchronize()
            evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
            for i in range(steps):
                flush.zero_()
                evs[i][0].record()
                env.step(acts[i % 16])
                evs[i][1].record()
            torch.cuda.synchronize()
            ms = sorted(a.elapsed_time(b) for a, b in evs)
            mean = sum(ms) / len(ms)
            print(json.dumps({
                "config": label, "scenario": name, "num_envs": B, "kwargs": kwargs,
                "mode": "cuda_graph" if graph else "eager", "steps": steps,
                "ms_per_step": round(mean, 4), "ms_median": round(ms[len(ms) // 2], 4),
                "ms_p90": round(ms[int(len(ms) * 0.9)], 4), "ms_max": round(ms[-1], 4),
                "env_steps_per_s": round(B / (mean * 1e-3), 1),
            }), flush=True)
            del env
    # host cost of one Environment.step: a tiny batch, so the GPU is never the limiter
    import time

    for label, name, _, kwargs in CONFIGS[:1] + CONFIGS[3:5]:
        env = b200.make_env(name, num_envs=32, device="cuda", seed=0, cuda_graph=True, **kwargs)
        env.reset()
        acts = [env.get_random_actions() for _ in range(16)]
        for i in range(20):
            env.step(acts[i % 16])
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(500):
            env.step(acts[i % 16])
        host = (time.perf_counter() - t0) / 500
        torch.cuda.synchronize()
        print(json.dumps({"config": label, "num_envs": 32, "mode": "cuda_graph", "host_us_per_step": round(host * 1e6, 1)}), flush=True)


main()
