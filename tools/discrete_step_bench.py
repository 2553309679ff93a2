"""The captured step of balance and transport3 per action space, with the action ingest inside the whole-step kernel
(one launch per step) and in a launch of its own in front of it (``_INGEST_IN_KERNEL = False``, two launches).

Each configuration is one ``cuda_graph=True`` env at 32768 envs: {continuous, discrete, multi-discrete} x
{prologue on, off}.  The envs of a workload are built side by side and their timed runs alternate (``--runs`` rounds),
so that drifting clocks and other tenants hit every configuration alike.  Timing as ``bench.py`` times its value:
CUDA events around every ``Environment.step`` with the L2 flushed outside the brackets.  Actions are pre-generated
on the device from a CPU generator (uniform in the range, or uniform indices).  The card's name, power limit and max
SM clock are read in the same process.  One JSON line per (workload, configuration, run), then a summary line per
workload with the median and the spread (max - min) of the runs.

    python tools/discrete_step_bench.py [--steps 300] [--warmup 20] [--runs 3] [--workloads balance,transport3]
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
SPACES = {"continuous": dict(), "discrete": dict(continuous_actions=False),
          "multidiscrete": dict(continuous_actions=False, multidiscrete_actions=True)}


def actions(env, steps, seed, device):
    """[steps][n_agents] device tensors in the env's action space."""
    gen = torch.Generator(device="cpu").manual_seed(seed)
    if env.continuous_actions:
        return bench.pregenerate_actions(env, steps, seed, device)
    out = []
    for _ in range(steps):
        per_agent = []
        for a in env.agents:
            nvec = a.discrete_action_nvec
            if env.multidiscrete_actions:
                k = torch.stack([torch.randint(0, n, (env.num_envs,), generator=gen) for n in nvec], -1)
            else:
                k = torch.randint(0, nvec[0] * nvec[1], (env.num_envs, 1), generator=gen)
            per_agent.append(k.to(device))
        out.append(per_agent)
    return out


class Arm:
    def __init__(self, config, n_envs, space, prologue, steps, warmup, device):
        import vectorizedmultiagentsimulator_b200 as b200
        from vectorizedmultiagentsimulator_b200.simulator.environment import environment as E

        cfg = bench.CONFIGS[config]
        saved = E._INGEST_IN_KERNEL, E._WHOLE_STEP_KERNEL_WAIT_S
        E._INGEST_IN_KERNEL, E._WHOLE_STEP_KERNEL_WAIT_S = prologue, 600.0  # (read when the step is captured)
        try:
            self.env = b200.make_env(cfg["scenario"], num_envs=n_envs, device=device, seed=0, cuda_graph=True,
                                     **SPACES[space], **cfg["kwargs"])
            self.acts = actions(self.env, warmup + steps, seed=1, device=device)
            for t in range(warmup):
                self.env.step(self.acts[t])
        finally:
            E._INGEST_IN_KERNEL, E._WHOLE_STEP_KERNEL_WAIT_S = saved
        plan = self.env._one_call
        self.one_kernel = bool(plan is not None and plan.c.fused_kernel > 0 and plan.c.ingest_in_kernel)
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
        raise SystemExit("discrete_step_bench.py measures on a CUDA device; none is visible")
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    gpu = card()
    flush = torch.empty(512 * 1024 * 1024, dtype=torch.uint8, device=device)
    for config in args.workloads.split(","):
        n = WORKLOADS[config]
        arms = {(space, on): Arm(config, n, space, on, args.steps, args.warmup, device)
                for space in SPACES for on in (True, False)}
        results = {key: [] for key in arms}
        for run in range(args.runs):
            for (space, on), arm in arms.items():
                ms = arm.value_ms(flush)
                results[(space, on)].append(ms)
                print(json.dumps({
                    "workload": config, "envs": n, "actions": space, "prologue": on, "run": run,
                    "us_per_step": round(ms * 1e3, 3), "launches_per_step": arm.launches_per_step,
                    "one_kernel": arm.one_kernel, "gpu": gpu,
                }), flush=True)
        summary = {
            f"{space}, prologue {'on' if on else 'off'}": {
                "median_us": round(statistics.median(v) * 1e3, 3), "spread_us": round((max(v) - min(v)) * 1e3, 3),
            }
            for (space, on), v in results.items()
        }
        print(json.dumps({"workload": config, "envs": n, "gpu": gpu, "summary": summary}), flush=True)
        del arms
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
