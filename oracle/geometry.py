"""ORACLE (test infrastructure, not product code) — closest-point geometry on CPU.

A plain torch-fp32 restatement of the reference's batched closest-point routines
(``vmas/simulator/physics.py``).  Every function is shape-generic: it works
on one pair (``[B, 2]``) or on a whole stacked bucket (``[B, P, 2]`` with per-pair lengths
``[P, 1]``), which is how ``oracle/world_step.py`` calls it.  Every function cites the
reference lines it follows.  Arithmetic order and fp32 scalar rounding follow the reference expression by
expression so that results are bit-comparable with it (checked in
``tests/test_oracle_vs_reference.py`` and pinned by ``tests/golden/``).

Conventions: points are ``[..., 2]``, angles ``[..., 1]``, lengths python floats (rounded to
fp32 here, as the reference does with ``torch.tensor``) or fp32 tensors ``[P, 1]``.
"""
from __future__ import annotations

import math

import torch

INF = float("inf")


def _len_t(length, like):
    """A python-float length as the fp32 tensor the reference builds with ``torch.tensor``.
    Tensors (one length per stacked pair, shape ``[P, 1]``) pass through."""
    if isinstance(length, torch.Tensor):
        return length
    return torch.tensor(length, dtype=torch.float32, device=like.device)


def unit(rot):
    """(cos, sin) of ``rot [B, 1]`` → ``[B, 2]`` (ref physics.py:413)."""
    return torch.cat([rot.cos(), rot.sin()], dim=-1)


def cross2(a, b):
    """Scalar 2-D cross product, ``[B, 1]`` (ref utils.py:194-197)."""
    return (a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]).unsqueeze(-1)


def closest_point_line(line_pos, line_rot, line_length, q, limit_to_line_length=True):
    """Closest point of a segment (centre, angle, length) to ``q`` (ref physics.py:400-429)."""
    direction = unit(line_rot)
    delta = line_pos - q
    along = (delta * direction).sum(-1).unsqueeze(-1)
    side = torch.sign(along)
    if limit_to_line_length:
        half = (_len_t(line_length, line_pos) / 2).expand(along.shape)
        reach = torch.minimum(torch.abs(along), half)
    else:
        reach = torch.abs(along)
    return line_pos - side * reach * direction


def line_extrema(line_pos, line_rot, line_length):
    """Both end points of a segment (ref physics.py:132-141)."""
    half = _len_t(line_length, line_pos) / 2
    offset = torch.cat([half * torch.cos(line_rot), half * torch.sin(line_rot)], dim=-1)
    return line_pos + offset, line_pos - offset


def intersection_line_line(a1, a2, b1, b2):
    """Segment/segment intersection point and a hit mask (ref physics.py:222-260)."""
    r = a2 - a1
    s = b2 - b1
    qp = b1 - a1
    qp_x_r = cross2(qp, r)
    qp_x_s = cross2(qp, s)
    r_x_s = cross2(r, s)
    u = qp_x_r / r_x_s
    t = qp_x_s / r_x_s
    hit = (~(r_x_s == 0)) & (0 <= u) & (u <= 1) & (0 <= t) & (t <= 1)
    point = torch.where(hit.expand(a1.shape), a1 + t * r, torch.full_like(a1, INF))
    return point, hit


def _first_minimum(candidates):
    """Strict-``<`` running minimum over (p1, p2) candidates (ref physics.py:207-213)."""
    p1_best = torch.full_like(candidates[0][0], INF)
    p2_best = torch.full_like(candidates[0][1], INF)
    d_best = torch.full(candidates[0][0].shape[:-1], INF, dtype=torch.float32, device=p1_best.device)
    for p1, p2 in candidates:
        d = torch.linalg.vector_norm(p1 - p2, dim=-1)
        better = d < d_best
        sel = better.unsqueeze(-1).expand(p1.shape)
        p1_best = torch.where(sel, p1, p1_best)
        p2_best = torch.where(sel, p2, p2_best)
        d_best = torch.where(better, d, d_best)
    return p1_best, p2_best


def closest_points_line_line(pos1, rot1, len1, pos2, rot2, len2):
    """Closest pair of points between two segments (ref physics.py:144-219)."""
    a1, a2 = line_extrema(pos1, rot1, len1)
    b1, b2 = line_extrema(pos2, rot2, len2)
    cross_point, hit = intersection_line_line(a1, a2, b1, b2)
    candidates = [
        (a1, closest_point_line(pos2, rot2, len2, a1)),
        (a2, closest_point_line(pos2, rot2, len2, a2)),
        (closest_point_line(pos1, rot1, len1, b1), b1),
        (closest_point_line(pos1, rot1, len1, b2), b2),
    ]
    p1, p2 = _first_minimum(candidates)
    sel = hit.expand(p1.shape)
    return torch.where(sel, cross_point, p1), torch.where(sel, cross_point, p2)


def box_sides(box_pos, box_rot, box_length, box_width):
    """The four sides of a box as (centre, angle, length) segments (ref physics.py:298-325)."""
    u = unit(box_rot)
    rot_perp = box_rot + torch.pi / 2
    v = unit(rot_perp)
    half_l = _len_t(box_length, box_pos) / 2
    half_w = _len_t(box_width, box_pos) / 2
    return [
        (box_pos + u * half_l, rot_perp, box_width),
        (box_pos - u * half_l, rot_perp, box_width),
        (box_pos + v * half_w, box_rot, box_length),
        (box_pos - v * half_w, box_rot, box_length),
    ]


def closest_point_box(box_pos, box_rot, box_length, box_width, q):
    """Closest point on a box outline to ``q`` (ref physics.py:263-295, 385-397)."""
    best = torch.full_like(box_pos, INF)
    d_best = torch.full(box_pos.shape[:-1], INF, dtype=torch.float32, device=box_pos.device)
    for pos, rot, length in box_sides(box_pos, box_rot, box_length, box_width):
        p = closest_point_line(pos, rot, length, q)
        d = torch.linalg.vector_norm(q - p, dim=-1)
        better = d < d_best
        best = torch.where(better.unsqueeze(-1).expand(p.shape), p, best)
        d_best = torch.where(better, d, d_best)
    return best


def closest_line_box(box_pos, box_rot, box_length, box_width, line_pos, line_rot, line_length):
    """Closest (point on box, point on line) (ref physics.py:328-382)."""
    candidates = [
        closest_points_line_line(pos, rot, length, line_pos, line_rot, line_length)
        for pos, rot, length in box_sides(box_pos, box_rot, box_length, box_width)
    ]
    return _first_minimum(candidates)


def closest_box_box(pos1, rot1, len1, wid1, pos2, rot2, len2, wid2):
    """Closest (point on box 1, point on box 2) (ref physics.py:26-129)."""
    candidates = []
    for pos, rot, length in box_sides(pos1, rot1, len1, wid1):
        on_box2, on_side = closest_line_box(pos2, rot2, len2, wid2, pos, rot, length)
        candidates.append((on_side, on_box2))
    for pos, rot, length in box_sides(pos2, rot2, len2, wid2):
        on_box1, on_side = closest_line_box(pos1, rot1, len1, wid1, pos, rot, length)
        candidates.append((on_box1, on_side))
    return _first_minimum(candidates)


def inner_point_box(outside, surface, box_pos):
    """Projection of the box centre on the approach direction (ref physics.py:13-23).

    Returns the point *inside* a solid box that contact forces are measured from and its
    depth.  When ``outside`` coincides with ``surface`` the reference returns
    ``2 * surface`` (depth 0); that quirk is kept.
    """
    v = surface - outside
    u = box_pos - surface
    v_norm = torch.linalg.vector_norm(v, dim=-1).unsqueeze(-1)
    depth = (v * u).sum(-1).unsqueeze(-1) / v_norm
    x = (v / v_norm) * depth
    degenerate = v_norm == 0
    x = torch.where(degenerate.expand(x.shape), surface, x)
    depth = torch.where(degenerate, 0, depth)
    return surface + x, torch.abs(depth.squeeze(-1))


HALF_PI = math.pi / 2
