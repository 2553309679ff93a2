"""Joints: distance / rotation constraints between two entities (ref vmas/simulator/joints.py).

A joint with ``dist > 0`` inserts a Line (or Box, when ``width > 0``) landmark between its two
end points and two zero-length constraints tying the landmark's ends to the entities; a joint
with ``dist == 0`` is a single constraint.  The constraint forces themselves are evaluated by
the CUDA substep kernel (``K_JOINT`` work items); this module only owns the static anchors and
the per-env ``fixed_rotation`` values the kernel reads.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch

from . import core as _core
from .utils import Color, Observer, TorchUtils, X, Y


def _check_anchor(anchor):
    assert (
        max(anchor) <= 1 and min(anchor) >= -1
    ), f"Joint anchor points should be between -1 and 1, got {anchor}"


def _check_pair(entity_a, entity_b, anchor_a, anchor_b, dist):
    assert entity_a != entity_b, "Cannot join same entity"
    _check_anchor(anchor_a)
    _check_anchor(anchor_b)
    assert dist >= 0, f"Joint dist must be >= 0, got {dist}"


class Joint(Observer):
    """User-facing joint.  ``dist == 0`` pins the two anchors together with one constraint;
    ``dist > 0`` spawns a movable link landmark (a Line, or a Box when ``width > 0``) whose two ends
    are pinned to the entities' anchors, and keeps it placed between them whenever an end point is
    repositioned through the state API (observer protocol)."""

    def __init__(
        self,
        entity_a,
        entity_b,
        anchor_a: Tuple[float, float] = (0.0, 0.0),
        anchor_b: Tuple[float, float] = (0.0, 0.0),
        rotate_a: bool = True,
        rotate_b: bool = True,
        dist: float = 0.0,
        collidable: bool = False,
        width: float = 0.0,
        mass: float = 1.0,
        fixed_rotation_a: Optional[float] = None,
        fixed_rotation_b: Optional[float] = None,
    ):
        _check_pair(entity_a, entity_b, anchor_a, anchor_b, dist)
        pinned = dist == 0
        if pinned:
            assert not collidable, "Cannot have collidable joint with dist 0"
            assert width == 0, "Cannot have width for joint with dist 0"
            assert (
                fixed_rotation_a == fixed_rotation_b
            ), "If dist is 0, fixed_rotation_a and fixed_rotation_b should be the same"
        for fixed, free, side in ((fixed_rotation_a, rotate_a, "a"), (fixed_rotation_b, rotate_b, "b")):
            if fixed is not None:
                assert not free, f"If you provide a fixed rotation for {side}, rotate_{side} should be False"
        if width > 0:
            assert collidable

        self.entity_a, self.entity_b = entity_a, entity_b
        self.rotate_a, self.rotate_b = rotate_a, rotate_b
        self.fixed_rotation_a, self.fixed_rotation_b = fixed_rotation_a, fixed_rotation_b
        self.landmark = None

        if pinned:
            self.joint_constraints = [
                JointConstraint(
                    entity_a,
                    entity_b,
                    anchor_a=anchor_a,
                    anchor_b=anchor_b,
                    dist=dist,
                    rotate=rotate_a and rotate_b,
                    fixed_rotation=fixed_rotation_a,
                )
            ]
            return

        for end in (entity_a, entity_b):
            end.subscribe(self)
        self.landmark = _core.Landmark(
            name=f"joint {entity_a.name} {entity_b.name}",
            collide=collidable,
            movable=True,
            rotatable=True,
            mass=mass,
            shape=_core.Box(length=dist, width=width) if width != 0 else _core.Line(length=dist),
            color=Color.BLACK,
            is_joint=True,
        )
        ends = (
            ((-1, 0), entity_a, anchor_a, rotate_a, fixed_rotation_a),
            ((1, 0), entity_b, anchor_b, rotate_b, fixed_rotation_b),
        )
        self.joint_constraints = [
            JointConstraint(
                self.landmark, entity, anchor_a=link_end, anchor_b=anchor, dist=0.0, rotate=free, fixed_rotation=fixed
            )
            for link_end, entity, anchor, free, fixed in ends
        ]

    def notify(self, observable, *args, **kwargs):
        """An end point was re-placed: put the link landmark between the two anchors again."""
        end_a = self.joint_constraints[0].pos_point(self.entity_a)
        end_b = self.joint_constraints[1].pos_point(self.entity_b)
        self.landmark.set_pos((end_a + end_b) / 2, batch_index=None)
        heading = torch.atan2(end_b[:, Y] - end_a[:, Y], end_b[:, X] - end_a[:, X]).unsqueeze(-1)
        self.landmark.set_rot(heading, batch_index=None)
        # a non-rotating end without an explicit angle keeps whatever angle it has now
        if not self.rotate_a and self.fixed_rotation_a is None:
            self.joint_constraints[0].fixed_rotation = heading - self.entity_a.state.rot
        if not self.rotate_b and self.fixed_rotation_b is None:
            self.joint_constraints[1].fixed_rotation = heading - self.entity_b.state.rot


class JointConstraint:
    """Uncollidable constraint tying two anchor points at a given distance (private)."""

    def __init__(
        self,
        entity_a,
        entity_b,
        anchor_a: Tuple[float, float] = (0.0, 0.0),
        anchor_b: Tuple[float, float] = (0.0, 0.0),
        dist: float = 0.0,
        rotate: bool = True,
        fixed_rotation: Optional[float] = None,
    ):
        _check_pair(entity_a, entity_b, anchor_a, anchor_b, dist)
        if fixed_rotation is not None:
            assert not rotate, "If fixed rotation is provided, rotate should be False"
        if rotate:
            assert fixed_rotation is None, "If you provide a fixed rotation, rotate should be False"
            fixed_rotation = 0.0

        self.entity_a = entity_a
        self.entity_b = entity_b
        self.anchor_a = anchor_a
        self.anchor_b = anchor_b
        self.dist = dist
        self.rotate = rotate
        self._fixed_rotation = fixed_rotation
        self._fixed_rotation_version = 0
        self._world = None
        self._anchor_delta_cache = {}

    @property
    def fixed_rotation(self):
        return self._fixed_rotation

    @fixed_rotation.setter
    def fixed_rotation(self, value):
        self._fixed_rotation = value
        self._fixed_rotation_version += 1  # the backend re-uploads this constraint's column

    def _delta_anchor_tensor(self, entity):
        if entity is self.entity_a:
            anchor = self.anchor_a
        elif entity is self.entity_b:
            anchor = self.anchor_b
        else:
            raise AssertionError()
        pos = entity.state.pos
        key = (id(entity), pos.device)
        t = self._anchor_delta_cache.get(key)
        if t is None:
            t = torch.tensor(
                entity.shape.get_delta_from_anchor(anchor), device=pos.device, dtype=torch.float32
            )
            self._anchor_delta_cache[key] = t
        return t.unsqueeze(0).expand(pos.shape)

    def get_delta_anchor(self, entity):
        return TorchUtils.rotate_vector(self._delta_anchor_tensor(entity), entity.state.rot)

    def pos_point(self, entity):
        return entity.state.pos + self.get_delta_anchor(entity)

    def render(self, env_index: int = 0):
        raise NotImplementedError("Rendering is outside the scope of the CUDA hot-path build")
