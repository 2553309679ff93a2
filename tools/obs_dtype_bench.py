"""fp32 vs 16-bit observations (``make_env(..., obs_dtype=...)``) on one GPU: ``bench.py``'s two arms per dtype.

* ``value``: the step's results stay in HBM; CUDA events around every ``Environment.step`` (L2 flushed outside
  the brackets), as ``bench.py`` times its value.
* ``e2e``: pinned host buffers, a copy stream and software pipelining, as ``bench.py``'s e2e arm: each bracket holds
  the step (its kernel reads the pinned actions where they lie) and the download of the previous step's
  observations, rewards and dones.  Also reported: the host's wall-clock time per pipelined step, and the time of
  one step's download alone (events around back-to-back downloads with nothing else running).

fp32, fp16 and bf16 envs of one workload are built side by side and their timed runs alternate (``--runs`` rounds),
so that drifting clocks and other tenants hit every dtype alike.  The D2H bytes per step are computed from the
shapes of what a step returns.  The card's name, power limit and max SM clock are read in the same process.  One
JSON line per (workload, dtype, run), then a summary line per workload.

    python tools/obs_dtype_bench.py [--steps 300] [--warmup 20] [--runs 2] [--workloads balance,transport3,navigation]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402

#: (bench.py config, envs): balance and transport3 at 32768 envs, navigation at 8192
WORKLOADS = {"balance": 32768, "transport3": 32768, "navigation": 8192}
DTYPES = {"fp32": torch.float32, "fp16": torch.float16, "bf16": torch.bfloat16}


def card():
    out = subprocess.run(
        ["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
        capture_output=True, text=True,
    )
    return out.stdout.strip() if out.returncode == 0 else f"nvidia-smi failed: {out.stderr.strip()}"


class Arm:
    """One env of a workload and its timed loops."""

    def __init__(self, config, n_envs, dtype, steps, warmup, device):
        import vectorizedmultiagentsimulator_b200 as b200

        cfg = bench.CONFIGS[config]
        self.env = b200.make_env(cfg["scenario"], num_envs=n_envs, device=device, seed=0, cuda_graph=True,
                                 obs_dtype=dtype, **cfg["kwargs"])
        self.steps, self.warmup, self.device = steps, warmup, device
        self.dev_actions = bench.pregenerate_actions(self.env, warmup + steps, seed=1, device=device)
        self.host_actions = bench.pregenerate_actions(self.env, warmup + steps, seed=101, device=device, pin=True)
        for t in range(warmup):
            self.env.step(self.dev_actions[t])
        obs, rew, done, _ = self.env.step(self.dev_actions[0])
        self.d2h_bytes = sum(t.numel() * t.element_size() for t in list(obs) + list(rew) + [done])
        self.host_sets = [
            (torch.empty((len(obs),) + tuple(obs[0].shape), dtype=obs[0].dtype).pin_memory(),
             torch.empty((len(rew),) + tuple(rew[0].shape), dtype=rew[0].dtype).pin_memory(),
             torch.empty(done.shape, dtype=done.dtype).pin_memory())
            for _ in range(2)
        ]
        self.copy_stream = torch.cuda.Stream(device=device)
        self.pending = None
        self.launches_per_step = None

    @staticmethod
    def _timed(fn, n, flush):
        pairs = []
        for i in range(n):
            if flush is not None:
                flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn(i)
            e1.record()
            pairs.append((e0, e1))
        torch.cuda.synchronize()
        return sum(a.elapsed_time(b) for a, b in pairs)

    def value_ms(self, flush):
        backend = self.env.world._get_backend()
        before = backend.launches
        W, acts = self.warmup, self.dev_actions
        ms = self._timed(lambda i: self.env.step(acts[W + i]), self.steps, flush)
        self.launches_per_step = (backend.launches - before) / self.steps
        return ms

    def _download(self, slot):
        main = torch.cuda.current_stream()
        self.copy_stream.wait_stream(main)
        with torch.cuda.stream(self.copy_stream):
            for dst, src in zip(self.host_sets[slot], self.pending):
                dst.copy_(src, non_blocking=True)

    def _e2e_step(self, i):
        import vectorizedmultiagentsimulator_b200 as b200

        main = torch.cuda.current_stream()
        actions = self.host_actions[(self.warmup + i) % len(self.host_actions)]
        if self.pending is not None:
            self._download(i & 1)
        obs, rews, dones, _ = self.env.step(actions)
        # (the per-agent results of a step sit back to back in one block: one view each, no stacking copy)
        fresh = (b200.stack_views(obs), b200.stack_views(rews), dones)
        main.wait_stream(self.copy_stream)  # the bracket closes after the download it overlapped
        self.pending = fresh

    def _download_and_wait(self, slot):
        self._download(slot)
        torch.cuda.current_stream().wait_stream(self.copy_stream)

    def download_ms(self, n=50):
        """One step's results to the pinned host buffers, alone on the link (mean of ``n``)."""
        import vectorizedmultiagentsimulator_b200 as b200

        obs, rews, dones, _ = self.env.step(self.dev_actions[0])
        self.pending = (b200.stack_views(obs), b200.stack_views(rews), dones)
        self.obs_one_view = self.pending[0].data_ptr() == obs[0].data_ptr()  # (no stacking copy in the e2e loop)
        torch.cuda.synchronize()
        ms = self._timed(lambda i: self._download_and_wait(i & 1), n, None)
        self.pending = None
        return ms / n

    def e2e_ms(self):
        import time

        self.pending = None
        for t in range(40):  # the first transfers after an idle link are slower
            self._e2e_step(t - self.warmup)
        torch.cuda.synchronize()
        wall0 = time.perf_counter()
        ms = self._timed(self._e2e_step, self.steps, None)
        self.wall_ms = (time.perf_counter() - wall0) * 1e3

        return ms + self._timed(lambda _: self._download_and_wait(0), 1, None)


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=300)
    p.add_argument("--warmup", type=int, default=20)
    p.add_argument("--runs", type=int, default=2)
    p.add_argument("--workloads", default=",".join(WORKLOADS))
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("obs_dtype_bench.py measures on a CUDA device; none is visible")
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    gpu = card()
    flush = torch.empty(512 * 1024 * 1024, dtype=torch.uint8, device=device)
    for config in args.workloads.split(","):
        n = WORKLOADS[config]
        arms = {label: Arm(config, n, dtype, args.steps, args.warmup, device) for label, dtype in DTYPES.items()}
        results = {label: [] for label in arms}
        for run in range(args.runs):
            for label, arm in arms.items():
                value = arm.value_ms(flush) / args.steps
                e2e = arm.e2e_ms() / args.steps
                download = arm.download_ms()
                row = {
                    "workload": config, "envs": n, "obs_dtype": label, "run": run,
                    "value_ms_per_step": round(value, 5), "value_env_steps_per_s": round(n / (value * 1e-3)),
                    "e2e_ms_per_step": round(e2e, 5), "e2e_env_steps_per_s": round(n / (e2e * 1e-3)),
                    "e2e_wall_ms_per_step": round(arm.wall_ms / args.steps, 5),
                    "download_alone_ms": round(download, 5), "download_gb_per_s": round(arm.d2h_bytes / download * 1e-6, 1),
                    "d2h_bytes_per_step": arm.d2h_bytes, "d2h_bytes_per_env_step": arm.d2h_bytes / n,
                    "launches_per_step": arm.launches_per_step, "obs_one_view": arm.obs_one_view, "gpu": gpu,
                }
                results[label].append(row)
                print(json.dumps(row), flush=True)
        summary = {
            label: {k: [r[k] for r in rows] for k in ("value_env_steps_per_s", "e2e_env_steps_per_s", "download_alone_ms")}
            | {"d2h_bytes_per_env_step": rows[0]["d2h_bytes_per_env_step"]}
            for label, rows in results.items()
        }
        print(json.dumps({"workload": config, "envs": n, "gpu": gpu, "summary": summary}), flush=True)
        del arms
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
