"""The captured step of balance and transport3 with a bounded episode: ``max_steps`` and ``terminated_truncated``
inside the whole-step kernel, against the same env without a limit and against the route such envs took before
(the captured graph replayed: ``_DIRECT_STEP = False``).

Each configuration is one ``cuda_graph=True`` env at 32768 envs with continuous actions: no limit; ``max_steps=200``;
``max_steps=200`` with ``terminated_truncated=True``; ``max_steps=200`` on the graph route.  The envs of a workload
are built side by side and their timed runs alternate (``--runs`` rounds), so that drifting clocks and other tenants
hit every configuration alike.  Timing as ``bench.py`` times its value: CUDA events around every ``Environment.step``
with the L2 flushed outside the brackets.  The card's name, power limit and max SM clock are read in the same
process.  One JSON line per (workload, configuration, run), then a summary line per workload with the median and the
spread (max - min) of the runs.

    python tools/episode_step_bench.py [--steps 300] [--warmup 20] [--runs 3] [--workloads balance,transport3]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402
from obs_dtype_bench import card  # noqa: E402

WORKLOADS = {"balance": 32768, "transport3": 32768}
#: label -> (Environment kwargs, module flags read when the step is captured)
CONFIGS = {
    "no limit": (dict(), dict()),
    "max_steps=200": (dict(max_steps=200), dict()),
    "max_steps=200, terminated_truncated": (dict(max_steps=200, terminated_truncated=True), dict()),
    "max_steps=200, graph route": (dict(max_steps=200), dict(_DIRECT_STEP=False)),
}


class Arm:
    def __init__(self, config, n_envs, label, steps, warmup, device):
        import vectorizedmultiagentsimulator_b200 as b200
        from vectorizedmultiagentsimulator_b200.simulator.environment import environment as E

        cfg = bench.CONFIGS[config]
        env_kw, flags = CONFIGS[label]
        flags = dict(flags, _WHOLE_STEP_KERNEL_WAIT_S=600.0)  # (a limit is part of the kernel: compiled at capture)
        saved = {k: getattr(E, k) for k in flags}
        for k, v in flags.items():
            setattr(E, k, v)
        try:
            self.env = b200.make_env(cfg["scenario"], num_envs=n_envs, device=device, seed=0, cuda_graph=True,
                                     **env_kw, **cfg["kwargs"])
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
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("episode_step_bench.py measures on a CUDA device; none is visible")
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    gpu = card()
    flush = torch.empty(512 * 1024 * 1024, dtype=torch.uint8, device=device)
    for config in args.workloads.split(","):
        n = WORKLOADS[config]
        arms = {label: Arm(config, n, label, args.steps, args.warmup, device) for label in CONFIGS}
        results = {label: [] for label in arms}
        for run in range(args.runs):
            for label, arm in arms.items():
                ms = arm.value_ms(flush)
                results[label].append(ms)
                print(json.dumps({
                    "workload": config, "envs": n, "config": label, "run": run, "us_per_step": round(ms * 1e3, 3),
                    "launches_per_step": arm.launches_per_step, "one_kernel": arm.one_kernel, "gpu": gpu,
                }), flush=True)
        summary = {
            label: {"median_us": round(statistics.median(v) * 1e3, 3), "spread_us": round((max(v) - min(v)) * 1e3, 3)}
            for label, v in results.items()
        }
        print(json.dumps({"workload": config, "envs": n, "gpu": gpu, "summary": summary}), flush=True)
        del arms
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
