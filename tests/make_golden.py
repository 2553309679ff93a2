"""Generates the golden fixtures under tests/golden/ from the UNMODIFIED reference.

Run with ``VMAS_REF`` pointing at a checkout of the reference (VMAS 1.5.2):

    VMAS_REF=/path/to/VectorizedMultiAgentSimulator python tests/make_golden.py

For every scenario below the reference is rolled out on CPU with seeded random actions and,
per step, the exact inputs of ``World.step`` (state slab incl. the processed action forces,
per-env joint rotations) and its outputs are recorded, together with the world description
(``plan.describe_world`` of the *reference* world), LIDAR measurements and a sample of
distance / overlap queries.  The tests read only the fixtures, never the reference.
"""
import itertools
import os
import random
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

import golden_pack  # noqa: E402
from refutil import import_reference, per_env_fixed_rotations, post_step, pre_step, world_state  # noqa: E402

from vectorizedmultiagentsimulator_b200.simulator import plan as P  # noqa: E402

# name, kwargs, num_envs, steps
CASES = [
    ("balance", dict(n_agents=4), 64, 100),  # BASELINE.json configs[0] (PR1 reference case)
    ("transport", dict(n_agents=4), 32, 25),
    ("navigation", dict(n_agents=8), 32, 25),
    ("flocking", dict(n_agents=5), 32, 25),
    ("pollock", dict(lidar=True), 8, 12),
    ("waterfall", dict(), 16, 20),
    ("reverse_transport", dict(), 16, 20),
    ("joint_passage", dict(), 16, 20),
    ("multi_give_way", dict(), 16, 20),
    ("give_way", dict(), 16, 20),
    ("wheel", dict(), 16, 20),
    ("dropout", dict(), 16, 15),
    ("wind_flocking", dict(), 16, 15),  # per-env gravity tensors (Entity.gravity as [B, 2])
    ("football", dict(), 8, 10),
    ("passage", dict(), 16, 15),
    # crafted worlds (tests/crafted.py) for the branches no reference scenario takes
    ("crafted_clamps", dict(), 33, 12),  # max_f / f_range / max_t / t_range, angular + linear friction
    ("crafted_joints_apart", dict(), 16, 4),  # joints with anchors clearly apart (strict-tolerance joint test)
    ("crafted_lonely", dict(), 1, 6),  # batch_dim = 1, no work item
    ("crafted_crowd", dict(), 4, 6),  # 70 entities
]


def record(vmas, name, kwargs, num_envs, steps):
    scenario = name
    if name.startswith("crafted_"):
        import crafted

        scenario = crafted.make_scenario("vmas", name[len("crafted_"):])
    env = vmas.make_env(scenario, num_envs=num_envs, device="cpu", seed=0, **kwargs)
    world = env.world
    desc = P.describe_world(world)
    fix = dict(name=name, kwargs=kwargs, desc=desc.to_json(), steps=[], lidar=[], queries=[])
    gen = torch.Generator().manual_seed(1)
    idx = {id(e): i for i, e in enumerate(world.entities)}
    prev_out = None
    for t in range(steps):
        actions = [
            (torch.rand(num_envs, a.action_size, generator=gen) * 2 - 1) * a.action.u_range_tensor
            for a in env.agents
        ]
        pre_step(env, actions)
        state_in = world_state(world)
        fixed = per_env_fixed_rotations(world, desc)
        gravity = {
            i: e.gravity.clone() for i, e in enumerate(world.entities) if desc.entities[i].get("gravity_per_env")
        }
        world.step()
        state_out = world_state(world)
        entry = dict(force=state_in["force"], torque=state_in["torque"], out=state_out)
        same = prev_out is not None and all(
            torch.equal(state_in[k], prev_out[k]) for k in ("pos", "vel", "rot", "ang_vel")
        )
        if not same:
            entry["state_in"] = {k: state_in[k] for k in ("pos", "vel", "rot", "ang_vel")}
        if fixed:
            entry["fixed_rot"] = fixed
        if gravity:
            entry["ent_gravity"] = gravity
        fix["steps"].append(entry)
        prev_out = state_out
        obs, rews, dones, infos = post_step(env)
        if t < 3 or t == steps - 1:
            entry["obs"] = [o.clone() for o in obs]
            entry["rews"] = [r.clone() for r in rews]
            entry["dones"] = dones.clone()
        # LIDAR: every sensor of every agent on the post-step state
        if t % 3 == 0:
            for a in world.agents:
                for s in a.sensors:
                    targets = [i for i, e in enumerate(world.entities) if e is not a and s.entity_filter(e)]
                    fix["lidar"].append(
                        dict(
                            step=t,
                            src=idx[id(a)],
                            targets=targets,
                            angles=s._angles.clone(),
                            max_range=float(s._max_range),
                            out=s.measure().clone(),
                        )
                    )
    # distance / overlap queries on the final state
    ents = world.entities
    rnd = random.Random(0)
    pairs = list(itertools.permutations(range(len(ents)), 2))
    rnd.shuffle(pairs)
    final = world_state(world)
    fix["final_state"] = final
    for a, b in pairs[:60]:
        pt = torch.randn(num_envs, 2, generator=gen)
        fix["queries"].append(
            dict(
                a=a,
                b=b,
                distance=world.get_distance(ents[a], ents[b]).clone(),
                overlap=world.is_overlapping(ents[a], ents[b]).clone(),
                point=pt,
                point_distance=world.get_distance_from_point(ents[a], pt).clone(),
            )
        )
    return fix


def _flatten(x):
    if isinstance(x, dict):
        return [v for k in sorted(x) for v in _flatten(x[k])]
    if isinstance(x, (list, tuple)):
        return [v for item in x for v in _flatten(item)]
    return [x]


def _leaves(x):
    return [t.clone() for t in _flatten(x)]


def record_env(vmas):
    """What the reference's ``Environment`` returned in tests/test_env_vs_reference.py's roll-outs, by case."""
    import crafted
    import stock_style
    from test_env_vs_reference import CASES as ENV_CASES

    fix = {}
    for name, kwargs in ENV_CASES:
        for continuous in (True, False):
            n_envs = 12
            env = vmas.make_env(name, num_envs=n_envs, device="cpu", seed=3, continuous_actions=continuous, **kwargs)
            rec = dict(reset=_leaves(env.reset(seed=5)), steps=[])
            gen = torch.Generator().manual_seed(11)
            for t in range(12):
                if continuous:
                    actions = [
                        (torch.rand(n_envs, a.action_size, generator=gen) * 2 - 1) * a.action.u_range_tensor
                        for a in env.agents
                    ]
                else:
                    actions = [torch.randint(0, 9, (n_envs, 1), generator=gen) for _ in env.agents]
                rec["steps"].append([_leaves(part) for part in env.step(actions)])
                if t == 5:
                    rec["reset_at"] = _leaves(env.reset_at(2))
            fix[f"{name}-{'continuous' if continuous else 'discrete'}"] = rec

    n_envs = 10
    env = vmas.make_env(stock_style.make_scenario("vmas"), num_envs=n_envs, device="cpu", seed=1, n_agents=3)
    rec = dict(steps=[])
    gen = torch.Generator().manual_seed(2)
    for t in range(10):
        actions = [(torch.rand(n_envs, a.action_size, generator=gen) * 2 - 1) for a in env.agents]
        rec["steps"].append([_leaves(part) for part in env.step(actions)])
        if t == 4:
            rec["reset_at"] = _leaves(env.reset_at(3))
    fix["stock_style"] = rec

    n_envs = 9
    env = vmas.make_env(crafted.make_scenario("vmas", "dynamics_zoo"), num_envs=n_envs, device="cpu", seed=2)
    rec = dict(steps=[])
    gen = torch.Generator().manual_seed(3)
    for t in range(8):
        actions = [(torch.rand(n_envs, a.action_size, generator=gen) * 2 - 1) * a.action.u_range_tensor for a in env.agents]
        obs = env.step(actions)[0]
        rec["steps"].append(
            dict(
                obs=_leaves(obs),
                force=[a.state.force.clone() for a in env.agents],
                torque=[a.state.torque.clone() for a in env.agents],
            )
        )
    fix["dynamics_zoo"] = rec

    env = vmas.make_env("balance", num_envs=4, device="cpu", seed=0, n_agents=3)
    env.seed(1)
    fix["spaces"] = dict(
        n_action_spaces=len(env.action_space.spaces),
        observation_shape=tuple(env.observation_space.spaces[0].shape),
        random_actions=_leaves(env.get_random_actions()),
    )
    return fix


def record_teacher_forced(vmas):
    """tests/test_oracle_vs_reference.py's cases: per step what the reference's ``World.step`` received and
    returned, every sensor's LIDAR reading every 4th step and distance / overlap queries on the final state."""
    import crafted
    from test_oracle_vs_reference import CASES as TF_CASES
    from test_oracle_vs_reference import case_id

    fix = {}
    for i, (name, kwargs, num_envs, steps, seed) in enumerate(TF_CASES):
        scenario = name
        if name.startswith("crafted_"):
            scenario = crafted.make_scenario("vmas", name[len("crafted_"):], seed=1000 + seed)
        env = vmas.make_env(scenario, num_envs=num_envs, device="cpu", seed=seed, **kwargs)
        world = env.world
        desc = P.describe_world(world)
        ents = world.entities
        gen = torch.Generator().manual_seed(100 + seed)
        rec = dict(desc=desc.to_json(), steps=[], lidar=[], queries=[])
        for t in range(steps):
            actions = [
                (torch.rand(num_envs, a.action_size, generator=gen) * 2 - 1) * a.action.u_range_tensor for a in env.agents
            ]
            pre_step(env, actions)
            state = world_state(world)
            fixed_rot = per_env_fixed_rotations(world, desc)
            gravity = {k: e.gravity.clone() for k, e in enumerate(ents) if desc.entities[k].get("gravity_per_env")}
            world.step()
            want = world_state(world)
            entry = dict(force=state["force"], torque=state["torque"], fixed_rot=fixed_rot, ent_gravity=gravity, out=want)
            prev = rec["steps"][-1]["out"] if rec["steps"] else None
            if prev is None or not all(torch.equal(state[k], prev[k]) for k in ("pos", "vel", "rot", "ang_vel")):
                entry["state_in"] = {k: state[k] for k in ("pos", "vel", "rot", "ang_vel")}  # else: the last out
            rec["steps"].append(entry)
            post_step(env)
            if t % 4 == 0:
                for k, a in enumerate(ents):
                    for s in getattr(a, "sensors", None) or []:
                        targets = [j for j, e in enumerate(ents) if e is not a and s.entity_filter(e)]
                        rec["lidar"].append(
                            dict(
                                step=t, src=k, targets=targets, angles=(s._angles + want["rot"][:, k].unsqueeze(-1)).clone(),
                                max_range=float(s._max_range), out=s.measure().clone(),
                            )
                        )
        final = world_state(world)
        rec["final_state"] = final
        for a, b in list(itertools.permutations(range(len(ents)), 2))[:40]:
            point = torch.randn(num_envs, 2, generator=gen)
            rec["queries"].append(
                dict(
                    a=a, b=b, distance=world.get_distance(ents[a], ents[b]).clone(),
                    overlap=world.is_overlapping(ents[a], ents[b]).clone(), point=point,
                    point_distance=world.get_distance_from_point(ents[a], point).clone(),
                )
            )
        fix[case_id(i, name)] = rec
    return fix


def record_spawn_sampler(vmas):
    """Positions drawn by the reference's ``ScenarioUtils.spawn_entities_randomly`` (tests/test_reset_oracle.py)."""
    from vmas.simulator.core import Landmark, Sphere, World
    from vmas.simulator.utils import ScenarioUtils

    B, n = 4000, 4
    torch.manual_seed(0)
    world = World(B, "cpu")
    ents = [Landmark(name=f"l{i}", shape=Sphere(0.05)) for i in range(n)]
    for e in ents:
        world.add_landmark(e)
    occ = torch.tensor([[[0.0, 0.0]]]).expand(B, 1, 2)
    ScenarioUtils.spawn_entities_randomly(ents, world, None, 0.5, (-1, 1), (-1, 1), occupied_positions=occ)
    return torch.stack([e.state.pos for e in ents], dim=1).numpy()


#: fixtures of the tests that compare with the reference's own results, under golden/reference/: a directory
#: of one ``golden_pack`` file per case, or one ``.npy`` file -> recorder
REFERENCE_FIXTURES = {
    "env": record_env,
    "teacher_forced": record_teacher_forced,
    "spawn_sampler.npy": record_spawn_sampler,
}


def main():
    import numpy as np

    vmas = import_reference()
    out_dir = os.path.join(HERE, "golden")
    os.makedirs(out_dir, exist_ok=True)
    regenerate = "--all" in sys.argv  # fixtures are append-only; pass --all to regenerate everything
    for name, kwargs, num_envs, steps in CASES:
        path = os.path.join(out_dir, f"{name}.pt")
        if os.path.exists(path) and not regenerate:
            continue
        fix = record(vmas, name, kwargs, num_envs, steps)
        torch.save(fix, path)
        print(f"{name:20s} B={num_envs:3d} T={steps:3d} lidar={len(fix['lidar']):3d} -> {os.path.getsize(path)/1e6:.2f} MB")
    os.makedirs(os.path.join(out_dir, "reference"), exist_ok=True)
    for file, recorder in REFERENCE_FIXTURES.items():
        path = os.path.join(out_dir, "reference", file)
        if os.path.exists(path) and not regenerate:
            continue
        fix = recorder(vmas)
        if file.endswith(".npy"):
            np.save(path, fix)
            print(f"{file:28s} -> {os.path.getsize(path)/1e3:.1f} kB")
            continue
        os.makedirs(path, exist_ok=True)
        for case, rec in fix.items():
            # the host's vector ISA: the tests compare bit for bit on the same one (transcendentals may round
            # differently in the last place elsewhere)
            rec["cpu_capability"] = torch.backends.cpu.get_cpu_capability()
            golden_pack.save(os.path.join(path, case + ".npz"), rec)
            print(f"{file}/{case + '.npz':28s} -> {os.path.getsize(os.path.join(path, case + '.npz'))/1e3:.1f} kB")


if __name__ == "__main__":
    main()
