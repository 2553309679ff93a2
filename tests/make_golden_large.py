"""Records the reference roll-outs of the large crafted worlds (``tests/crafted_large.py``) for the tests.

    VMAS_REF=/path/to/VectorizedMultiAgentSimulator python tests/make_golden_large.py

Writes ``tests/golden/reference/teacher_forced/large_{160,520,1024}-{0,1,2}.npz``: per step what the
reference's ``World.step`` received — state, processed action forces, per-env joint rotations — and what it
returned.  Teacher-forced only: the ``tests/golden/*.pt`` roll-outs feed every golden-fixture test, including
the lane-per-entity mapping that stops at 128 entities.
"""
import os
import sys
import time

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import golden_pack  # noqa: E402
from refutil import import_reference, per_env_fixed_rotations, post_step, pre_step, world_state  # noqa: E402

from vectorizedmultiagentsimulator_b200.simulator import plan as P  # noqa: E402

# name, num_envs, steps, seed
CASES = [("large_160", 6, 5, 31), ("large_520", 4, 4, 32), ("large_1024", 4, 3, 33)]
STATE = ("pos", "vel", "rot", "ang_vel")


def case_id(i, name):
    return f"{name}-{i}"


def record(vmas, name, num_envs, steps, seed):
    import crafted_large

    env = vmas.make_env(crafted_large.make_scenario("vmas", name, seed=1000 + seed), num_envs=num_envs, device="cpu",
                        seed=seed)
    world = env.world
    t0 = time.perf_counter()
    desc = P.describe_world(world)
    print(f"{name}: describe_world {time.perf_counter() - t0:.2f} s, {len(desc.items)} work items")
    gen = torch.Generator().manual_seed(100 + seed)
    rec = dict(desc=desc.to_json(), steps=[])
    for t in range(steps):
        actions = [(torch.rand(num_envs, a.action_size, generator=gen) * 2 - 1) * a.action.u_range_tensor for a in env.agents]
        pre_step(env, actions)
        state = world_state(world)
        world.step()
        entry = dict(force=state["force"], torque=state["torque"], fixed_rot=per_env_fixed_rotations(world, desc),
                     ent_gravity={}, out=world_state(world))
        prev = rec["steps"][-1]["out"] if rec["steps"] else None
        if prev is None or not all(torch.equal(state[k], prev[k]) for k in STATE):
            entry["state_in"] = {k: state[k] for k in STATE}
        rec["steps"].append(entry)
        post_step(env)
    return rec


def main():
    vmas = import_reference()
    out_dir = os.path.join(HERE, "golden", "reference", "teacher_forced")
    os.makedirs(out_dir, exist_ok=True)
    for i, (name, num_envs, steps, seed) in enumerate(CASES):
        rec = record(vmas, name, num_envs, steps, seed)
        rec["cpu_capability"] = torch.backends.cpu.get_cpu_capability()
        path = os.path.join(out_dir, case_id(i, name) + ".npz")
        golden_pack.save(path, rec)
        print(f"{os.path.basename(path):28s} -> {os.path.getsize(path) / 1e3:.1f} kB")


if __name__ == "__main__":
    main()
