"""The captured step of a scenario whose observations read LIDARs: one kernel (the rays cast in the whole-step kernel's
epilogue) against the route such envs took before (the captured graph replayed: ``_DIRECT_STEP = False``, the rays
cast by ``cast_rays_batched_kernel``).

The two scenarios of tests/test_lidar_one_kernel_gpu.py: ``nav`` (navigation's world, 4 agents whose 12-ray LIDARs see
the other agents, 2 substeps, no masked pairs) and ``balance`` (balance with 4 agents whose 7-ray LIDARs see the
other agents, the package, the line and the floor; masked pairs, so the grid barrier), each at 8192 and 32768 envs
with continuous actions.  The envs of a workload are built side by side and their timed runs alternate (``--runs``
rounds), so that drifting clocks and other tenants hit every configuration alike.  Timing as ``bench.py`` times its
value: CUDA events around every ``Environment.step`` with the L2 flushed outside the brackets.  The card's name,
power limit and max SM clock are read in the same process.  One JSON line per (workload, envs, configuration, run),
then a summary line per (workload, envs) with the median and the spread (max - min) of the runs.

    python tools/lidar_step_bench.py [--steps 300] [--warmup 20] [--runs 3] [--workloads nav,balance] [--envs 8192,32768]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

import bench  # noqa: E402
from obs_dtype_bench import card  # noqa: E402
from test_lidar_one_kernel_gpu import LidarBalance, LidarNavigation  # noqa: E402

WORKLOADS = {"nav": (LidarNavigation, dict(n_agents=4)), "balance": (LidarBalance, dict(n_agents=4))}
#: label -> module flags read when the step is captured
CONFIGS = {"one kernel": dict(), "graph route": dict(_DIRECT_STEP=False)}


class Arm:
    def __init__(self, workload, n_envs, label, steps, warmup, device):
        import vectorizedmultiagentsimulator_b200 as b200
        from vectorizedmultiagentsimulator_b200.simulator.environment import environment as E

        cls, kwargs = WORKLOADS[workload]
        flags = dict(CONFIGS[label], _WHOLE_STEP_KERNEL_WAIT_S=600.0)  # (compiled at capture)
        saved = {k: getattr(E, k) for k in flags}
        for k, v in flags.items():
            setattr(E, k, v)
        try:
            self.env = b200.make_env(cls(), num_envs=n_envs, device=device, seed=0, cuda_graph=True, **kwargs)
            self.acts = bench.pregenerate_actions(self.env, warmup + steps, 1, device)
            for t in range(warmup):
                self.env.step(self.acts[t])
        finally:
            for k, v in saved.items():
                setattr(E, k, v)
        plan = self.env._one_call
        self.one_kernel = bool(plan is not None and plan.direct and plan.c.fused_kernel > 0 and plan.c.ingest_in_kernel)
        self.steps, self.warmup = steps, warmup

    def value_ms(self, flush):
        backend = self.env.world._get_backend()
        before = backend.launches
        pairs = []
        for i in range(self.steps):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            self.env.step(self.acts[self.warmup + i])
            e1.record()
            pairs.append((e0, e1))
        torch.cuda.synchronize()
        self.launches_per_step = (backend.launches - before) / self.steps
        return sum(a.elapsed_time(b) for a, b in pairs) / self.steps


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=300)
    p.add_argument("--warmup", type=int, default=20)
    p.add_argument("--runs", type=int, default=3)
    p.add_argument("--workloads", default=",".join(WORKLOADS))
    p.add_argument("--envs", default="8192,32768")
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lidar_step_bench.py measures on a CUDA device; none is visible")
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    gpu = card()
    flush = torch.empty(512 * 1024 * 1024, dtype=torch.uint8, device=device)
    for workload in args.workloads.split(","):
        for n in (int(x) for x in args.envs.split(",")):
            arms = {label: Arm(workload, n, label, args.steps, args.warmup, device) for label in CONFIGS}
            results = {label: [] for label in arms}
            for run in range(args.runs):
                for label, arm in arms.items():
                    ms = arm.value_ms(flush)
                    results[label].append(ms)
                    print(json.dumps({
                        "workload": workload, "envs": n, "config": label, "run": run,
                        "us_per_step": round(ms * 1e3, 3), "launches_per_step": arm.launches_per_step,
                        "one_kernel": arm.one_kernel, "gpu": gpu,
                    }), flush=True)
            summary = {
                label: {"median_us": round(statistics.median(v) * 1e3, 3), "spread_us": round((max(v) - min(v)) * 1e3, 3)}
                for label, v in results.items()
            }
            print(json.dumps({"workload": workload, "envs": n, "gpu": gpu, "summary": summary}), flush=True)
            del arms
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
