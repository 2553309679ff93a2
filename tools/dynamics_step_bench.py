"""The captured step of balance (4 agents) with agents of each action model the one-kernel prologue runs, and of a
world mixing them, with the action ingest inside the whole-step kernel (one launch per step) and in a launch of its
own in front of it (``_INGEST_IN_KERNEL = False``, two launches).

Each configuration is one ``cuda_graph=True`` env at 32768 envs with continuous actions: {model} x {prologue on, off}.
The two envs of a model are built side by side and their timed runs alternate (``--runs`` rounds), so that drifting
clocks and other tenants hit both alike.  Timing as ``bench.py`` times its value: CUDA events around every
``Environment.step`` with the L2 flushed outside the brackets.  Actions are pre-generated on the device from a CPU
generator (uniform in each agent's range).  The card's name, power limit and max SM clock are read in the same process.
One JSON line per (model, configuration, run), then a summary line per model with the median and the spread
(max - min) of the runs.

    python tools/dynamics_step_bench.py [--steps 300] [--warmup 20] [--runs 3] [--models holo_rot,diff,...]
"""
import argparse
import json
import os
import statistics
import sys
from types import SimpleNamespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from obs_dtype_bench import card  # noqa: E402

N_ENVS = 32768
MODEL_DT = SimpleNamespace(dt=0.1)  # (what the kinematic models read of their world)


def models():
    from vectorizedmultiagentsimulator_b200.simulator.dynamics.basic import (
        Forward, Holonomic, HolonomicWithRotation, Rotation,
    )
    from vectorizedmultiagentsimulator_b200.simulator.dynamics.diff_drive import DiffDrive
    from vectorizedmultiagentsimulator_b200.simulator.dynamics.kinematic_bicycle import KinematicBicycle

    return {  # name: (dynamics factory, u_range)
        "holo": (Holonomic, [1.0, 1.0]),
        "holo_rot": (HolonomicWithRotation, [1.0, 0.8, 0.5]),
        "forward": (Forward, [1.2]),
        "rotation": (Rotation, [0.6]),
        "diff": (lambda: DiffDrive(MODEL_DT, integration="rk4"), [1.0, 1.5]),
        "bicycle": (lambda: KinematicBicycle(MODEL_DT, width=0.05, l_f=0.06, l_r=0.04, max_steering_angle=0.6),
                    [1.0, 0.8]),
    }


LINEUPS = {
    "holo_rot": ["holo_rot"], "forward": ["forward"], "rotation": ["rotation"], "diff": ["diff"],
    "bicycle": ["bicycle"], "mixed": ["holo_rot", "diff", "rotation", "forward"],
}


def scenario(lineup):
    """balance whose agents get the action models of ``lineup`` in turn (rotatable)."""
    from vectorizedmultiagentsimulator_b200.scenarios import balance

    table = models()

    class Scenario(balance.Scenario):
        def make_world(self, batch_dim, device, **kwargs):
            orig, count = balance.Agent, iter(range(1 << 20))

            def agent(**kw):
                factory, u_range = table[lineup[next(count) % len(lineup)]]
                kw.update(dynamics=factory(), u_range=u_range, rotatable=True)
                return orig(**kw)

            balance.Agent = agent
            try:
                return super().make_world(batch_dim, device, **kwargs)
            finally:
                balance.Agent = orig

    return Scenario()


def actions(env, steps, seed, device):
    """[steps][n_agents] fp32 device tensors, uniform in each agent's range."""
    gen = torch.Generator(device="cpu").manual_seed(seed)
    out = []
    for _ in range(steps):
        out.append([((torch.rand(env.num_envs, a.action_size, generator=gen) * 2 - 1)
                     * torch.tensor(a.action.u_range_tensor.tolist())).to(device) for a in env.agents])
    return out


class Arm:
    def __init__(self, lineup, prologue, steps, warmup, device):
        import vectorizedmultiagentsimulator_b200 as b200
        from vectorizedmultiagentsimulator_b200.simulator.environment import environment as E

        saved = E._INGEST_IN_KERNEL, E._WHOLE_STEP_KERNEL_WAIT_S
        E._INGEST_IN_KERNEL, E._WHOLE_STEP_KERNEL_WAIT_S = prologue, 600.0  # (read when the step is captured)
        try:
            self.env = b200.make_env(scenario(lineup), num_envs=N_ENVS, device=device, seed=0, cuda_graph=True,
                                     n_agents=4)
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
    p.add_argument("--models", default=",".join(LINEUPS))
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dynamics_step_bench.py measures on a CUDA device; none is visible")
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    gpu = card()
    flush = torch.empty(512 * 1024 * 1024, dtype=torch.uint8, device=device)
    for name in args.models.split(","):
        arms = {on: Arm(LINEUPS[name], on, args.steps, args.warmup, device) for on in (True, False)}
        results = {on: [] for on in arms}
        for run in range(args.runs):
            for on, arm in arms.items():
                ms = arm.value_ms(flush)
                results[on].append(ms)
                print(json.dumps({
                    "workload": "balance", "agents": name, "envs": N_ENVS, "prologue": on, "run": run,
                    "us_per_step": round(ms * 1e3, 3), "launches_per_step": arm.launches_per_step,
                    "one_kernel": arm.one_kernel, "gpu": gpu,
                }), flush=True)
        summary = {
            f"prologue {'on' if on else 'off'}": {
                "median_us": round(statistics.median(v) * 1e3, 3), "spread_us": round((max(v) - min(v)) * 1e3, 3),
            }
            for on, v in results.items()
        }
        print(json.dumps({"workload": "balance", "agents": name, "envs": N_ENVS, "gpu": gpu, "summary": summary}),
              flush=True)
        del arms
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
