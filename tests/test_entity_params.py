"""Per-env entity mass and friction coefficients (domain randomisation) on the CPU: the oracle against the
reference's recorded roll-out, the host API (``Entity.mass`` / ``linear_friction`` / ``angular_friction`` as
``[batch_dim, 1]`` tensors), and the world hashes of every existing world."""
import os

import pytest
import torch

import crafted_params
import golden_pack
import param_oracle
from golden_util import GOLDEN_DIR
from vectorizedmultiagentsimulator_b200 import codegen
from vectorizedmultiagentsimulator_b200.simulator import plan as P
from vectorizedmultiagentsimulator_b200.simulator.core import Agent, Box, Landmark, Line, Sphere, World
from vectorizedmultiagentsimulator_b200.simulator.dynamics.diff_drive import DiffDrive

STATE = ("pos", "vel", "rot", "ang_vel")
FIXTURE = os.path.join(GOLDEN_DIR, "reference", "teacher_forced", "crafted_randomised-0.npz")

#: codegen.world_hash of every golden world's description, as the commit before per-env parameters computed it
PARENT_HASHES = {
    "balance": 0xE39178694E3E33D8,
    "crafted_clamps": 0xAA8CDF5CB787C498,
    "crafted_crowd": 0xE2D5420E9894C4E0,
    "crafted_joints_apart": 0x38089A218264465E,
    "crafted_lonely": 0x17459221CFCCC38D,
    "dropout": 0x3E5395D85DE1DEC0,
    "flocking": 0xCE48F2FF597017CF,
    "football": 0x33B34CD2567B118F,
    "give_way": 0x900B56922B1EEC7B,
    "joint_passage": 0xA9B96EE08878E8BF,
    "multi_give_way": 0xAB017B101B42778A,
    "navigation": 0x6443AD8E1B6117B5,
    "passage": 0xBB8B5AA676EBDAC4,
    "pollock": 0x854D2C77E4591657,
    "reverse_transport": 0x17BB052932DBB9E9,
    "transport": 0x0B085956A4DDBF69,
    "waterfall": 0xA9A334110240DEE3,
    "wheel": 0x5B343D661444A78B,
    "wind_flocking": 0x46071E08A62EFFE1,
    "balance-0": 0x15ADF49AC65B88F7,
    "balance-1": 0xA7B9E49CA3A575D1,
    "crafted_clamps-11": 0xAA8CDF5CB787C498,
    "crafted_crowd-14": 0xE2D5420E9894C4E0,
    "crafted_joints_apart-12": 0x38089A218264465E,
    "crafted_lonely-13": 0x17459221CFCCC38D,
    "flocking-4": 0x3E91893E0CE3849D,
    "joint_passage-8": 0xA9B96EE08878E8BF,
    "navigation-3": 0x94053FDBE3F9DB12,
    "pollock-5": 0x854D2C77E4591657,
    "reverse_transport-7": 0x17BB052932DBB9E9,
    "transport-2": 0xBBC22F4B72A4E565,
    "waterfall-6": 0xA9A334110240DEE3,
    "wheel-9": 0x5B343D661444A78B,
    "wind_flocking-10": 0x46071E08A62EFFE1,
}
#: the ahead-of-time specialisations' hashes (csrc/generated/specializations.cuh) of the commit before
PARENT_PRESET_HASHES = [
    0xE39178694E3E33D8, 0x15ADF49AC65B88F7, 0x0B085956A4DDBF69, 0x4AA0CD6CE3CA7B77,
    0x6443AD8E1B6117B5, 0x849CC8EAA9F56C3D, 0xCE48F2FF597017CF, 0x3E91893E0CE3849D,
]


def _stored_desc(name):
    if "-" in name:
        return golden_pack.load(os.path.join(GOLDEN_DIR, "reference", "teacher_forced", name + ".npz"))["desc"]
    return torch.load(os.path.join(GOLDEN_DIR, name + ".pt"), weights_only=False)["desc"]


# ---- world hashes --------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(PARENT_HASHES))
def test_world_hash_of_existing_worlds_unchanged(name):
    assert codegen.world_hash(P.WorldDescription.from_json(_stored_desc(name))) == PARENT_HASHES[name]


def test_preset_descriptions_hash_as_before():
    """Worlds described afresh (new description fields, false) hash as the parent described them."""
    hashes = [codegen.world_hash(desc) for _, desc, _ in codegen.preset_descriptions()]
    assert hashes == PARENT_PRESET_HASHES


def test_emitted_world_unchanged_without_per_env_parameters():
    """The generated header of the ahead-of-time worlds is what codegen emits (no per-env mask in it)."""
    for label, desc, tuning in codegen.preset_descriptions():
        _, text, _ = codegen.emit_world(desc, label, tuning)
        assert "PER_ENV" not in text


# ---- the oracle against the reference --------------------------------------------------------------------
def _same(got, want, rec):
    if rec["cpu_capability"] == torch.backends.cpu.get_cpu_capability():
        return torch.equal(got, want)
    return got.shape == want.shape and float((got - want).abs().max()) <= 2e-6


def test_fixture_has_per_env_parameters():
    rec = golden_pack.load(FIXTURE)
    desc = P.WorldDescription.from_json(rec["desc"])
    by_name = {e["name"]: e for e in desc.entities}
    for name, attrs in crafted_params.PER_ENV.items():
        e = by_name[name]
        assert e["mass_per_env"] == ("mass" in attrs)
        assert e["lin_fric_per_env"] == ("linear_friction" in attrs)
        assert e["ang_fric_per_env"] == ("angular_friction" in attrs)
        assert e["gravity_per_env"] == ("gravity" in attrs)
    kinds = {it["kind"] for it in desc.items}
    assert P.K_JOINT in kinds and {P.K_BS, P.K_LS, P.K_BL} <= kinds
    # the values change during the roll-out (re-drawn every few steps) and differ between envs
    m0 = [s["ent_params"][0]["mass"] for s in rec["steps"]]
    assert not torch.equal(m0[0], m0[-1]) and float(m0[0].std()) > 0


def test_oracle_equals_reference_bit_for_bit():
    rec = golden_pack.load(FIXTURE)
    tables = P.build_tables(P.WorldDescription.from_json(rec["desc"]))
    prev = None
    for t, entry in enumerate(rec["steps"]):
        state = {k: v.clone() for k, v in entry.get("state_in", prev).items() if k in STATE}
        state["force"], state["torque"] = entry["force"].clone(), entry["torque"].clone()
        param_oracle.world_step(
            tables, state, entry["ent_params"], fixed_rot=entry["fixed_rot"], ent_gravity=entry["ent_gravity"]
        )
        for k in STATE:
            want = entry["out"][k]
            assert _same(state[k], want, rec), f"step {t}: {k} max |diff| {float((state[k] - want).abs().max())}"
        prev = entry["out"]


# ---- host API ---------------------------------------------------------------------------------------------
def _world(B=4):
    world = World(B, "cpu", substeps=2)
    world.add_agent(Agent(name="a", shape=Sphere(0.05), rotatable=True))
    world.add_landmark(Landmark("box", shape=Box(0.2, 0.1), movable=True, rotatable=True))
    world.add_landmark(Landmark("bar", shape=Line(0.3), movable=True, rotatable=True))
    return world


def _hash(world):
    return codegen.world_hash(P.describe_world(world))


@pytest.mark.parametrize("attr", ["mass", "linear_friction", "angular_friction"])
def test_rejects_wrong_shape_dtype(attr):
    world = _world(4)
    a = world.agents[0]
    for bad in (torch.ones(4), torch.ones(4, 2), torch.ones(3, 1), torch.ones(4, 1, dtype=torch.float64)):
        with pytest.raises(ValueError, match=f"'a'.*{attr}"):
            setattr(a, attr, bad)
    with pytest.raises(ValueError, match=f"'b'.*{attr}"):
        Agent(name="b", **{attr: torch.ones(4, 1, dtype=torch.int32)})
    with pytest.raises(ValueError, match=f"'c'.*{attr}"):
        world.add_agent(Agent(name="c", **{attr: torch.ones(5, 1)}))


def test_rejects_wrong_device():
    world = _world(4)
    with pytest.raises(ValueError, match="'a'.*mass.*device"):
        world.agents[0].mass = torch.ones(4, 1, device="meta")


def test_kinematic_agent_rejects_per_env_mass():
    world = World(4, "cpu")
    world.add_agent(Agent(name="dd", shape=Sphere(0.05), rotatable=True, dynamics=DiffDrive(world), action_size=2))
    world.agents[0].mass = torch.ones(4, 1)
    with pytest.raises(NotImplementedError, match="'dd'.*out of scope"):
        P.describe_world(world)


def test_value_semantics_and_plan_version():
    world = _world(4)
    a, box = world.agents[0], world.landmarks[0]
    h0, v0 = _hash(world), world._plan_version
    # scalar -> tensor: structure (plan rebuilt, new hash)
    a.mass = torch.full((4, 1), 2.0)
    box.angular_friction = torch.full((4, 1), 0.1)
    a.linear_friction = torch.full((4, 1), 0.2)
    v1, h1 = world._plan_version, _hash(world)
    assert v1 > v0 and h1 != h0
    buf = a.mass
    # tensor -> tensor and in-place edits: data only
    fresh = torch.arange(4, dtype=torch.float32).unsqueeze(-1) + 1
    a.mass = fresh
    assert a.mass is buf and a.mass.data_ptr() == buf.data_ptr() and torch.equal(a.mass, fresh)
    fresh[0] = 99.0
    assert float(a.mass[0]) == 1.0  # (a copy, not an alias of the caller's tensor)
    a.mass[2] = 7.0
    box.angular_friction = torch.full((4, 1), 0.3)
    a.linear_friction[1] = 0.5
    assert world._plan_version == v1 and _hash(world) == h1
    # the moment of inertia follows the per-env mass (ref shape.moment_of_inertia(mass))
    assert torch.equal(a.moment_of_inertia, (1 / 2) * a.mass * a.shape.radius**2)
    # the values do not enter the hash
    world2 = _world(4)
    world2.agents[0].mass = torch.full((4, 1), 5.0)
    world2.landmarks[0].angular_friction = torch.full((4, 1), 0.9)
    world2.agents[0].linear_friction = torch.full((4, 1), 0.01)
    assert _hash(world2) == h1
    # tensor -> scalar: structure again, back to the original hash
    a.mass = 1.0
    box.angular_friction = None
    a.linear_friction = None
    assert world._plan_version > v1 and _hash(world) == h0


def test_description_flags_and_inertia_constants():
    world = _world(4)
    for e in world.entities:
        e.mass = torch.ones(4, 1)
    tables = P.build_tables(P.describe_world(world))
    for i, e in enumerate(tables.desc.entities):
        assert e["mass_per_env"] and e["mass"] == P.PER_ENV_PLACEHOLDER
        assert tables.ent_i32[i, 1] & P.F_MASS_ENV
    row = {e.name: tables.ent_f32[i] for i, e in enumerate(world.entities)}
    sphere, box, line = row["a"], row["box"], row["bar"]
    f32 = lambda x: float(torch.tensor(x, dtype=torch.float32))  # noqa: E731
    assert (sphere[P.EF_INERTIA_K0], sphere[P.EF_INERTIA_K1]) == (f32(1 / 2), f32(0.05**2))
    assert (box[P.EF_INERTIA_K0], box[P.EF_INERTIA_K1]) == (f32(1 / 12), f32(0.2**2 + 0.1**2))
    assert (line[P.EF_INERTIA_K0], line[P.EF_INERTIA_K1]) == (f32(1 / 12), f32(0.3**2))


def test_specialisable_and_whole_step_declined():
    from vectorizedmultiagentsimulator_b200 import jit

    desc = P.WorldDescription.from_json(golden_pack.load(FIXTURE)["desc"])
    assert codegen.specializable(desc, per_env=True) and codegen.has_per_env_params(desc)
    assert not codegen.specializable(desc)  # (what the whole-step kernels and the preset list ask)
    assert jit.request_step_kernel(desc, None, []) is None
    _, text, _ = codegen.emit_world(desc, "randomised")
    assert "PER_ENV" in text
    wind = P.WorldDescription.from_json(_stored_desc("wind_flocking"))
    assert codegen.specializable(wind, per_env=True) and codegen.has_per_env_params(wind)
