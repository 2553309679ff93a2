"""ORACLE (test infrastructure, not product code) — LIDAR ray casting and distance queries on CPU.

Torch-fp32 restatement of ``World.cast_rays`` and its three shape kernels
(``vmas/simulator/core.py:1281-1372, 1414-1490, 1544-1626, 1662-1786``) and of
``get_distance_from_point`` / ``get_distance`` / ``is_overlapping`` (core.py:1788-1969).
Pinned the same way as ``oracle/world_step.py`` (live reference comparison + golden fixtures).
"""
from __future__ import annotations

from typing import List

import torch

from vectorizedmultiagentsimulator_b200.simulator import plan as P
from vectorizedmultiagentsimulator_b200.simulator.utils import LINE_MIN_DIST

from . import geometry as G
from .world_step import rotate


def _rays_to_sphere(center, radius, origin, angles, max_range):
    """``center [B,2]``, ``origin [B,2]``, ``angles [B,R]`` → ``[B,R]`` (ref core.py:1414-1490)."""
    B, R = angles.shape
    o = origin.unsqueeze(1).expand(B, R, 2)
    c = center.unsqueeze(1).expand(B, R, 2)
    direction = torch.stack([torch.cos(angles), torch.sin(angles)], dim=-1)
    line_pos = o + direction * (max_range / 2)
    closest = G.closest_point_line(line_pos, angles.unsqueeze(-1), max_range, c, limit_to_line_length=False)
    d_norm = torch.linalg.vector_norm(c - closest, dim=-1)
    r = torch.tensor(radius, dtype=torch.float32)
    intersects = d_norm < r
    a = r**2 - d_norm**2
    m = torch.sqrt(torch.where(a > 0, a, 1e-8))
    in_front = ((c - o) * direction).sum(-1) > 0.0
    dist = torch.linalg.vector_norm(closest - o, dim=-1) - m
    return torch.where(intersects & in_front, dist, torch.full_like(dist, max_range))


def _rays_to_box(center, box_rot, length, width, origin, angles, max_range):
    """Slab test in the box frame (ref core.py:1281-1372); ``box_rot [B,1]``."""
    B, R = angles.shape
    o = origin.unsqueeze(1).expand(B, R, 2)
    c = center.unsqueeze(1).expand(B, R, 2)
    rot = box_rot.expand(B, R)
    L = torch.tensor(length, dtype=torch.float32)
    W = torch.tensor(width, dtype=torch.float32)
    o_local = rotate(o - c, (-rot).unsqueeze(-1))
    d_world = torch.stack([torch.cos(angles), torch.sin(angles)], dim=-1)
    d_local = rotate(d_world, (-rot).unsqueeze(-1))
    tx1 = (-L / 2 - o_local[..., 0]) / d_local[..., 0]
    tx2 = (L / 2 - o_local[..., 0]) / d_local[..., 0]
    tmin = torch.min(torch.stack([tx1, tx2], dim=-1), dim=-1)[0]
    tmax = torch.max(torch.stack([tx1, tx2], dim=-1), dim=-1)[0]
    ty1 = (-W / 2 - o_local[..., 1]) / d_local[..., 1]
    ty2 = (W / 2 - o_local[..., 1]) / d_local[..., 1]
    tymin = torch.min(torch.stack([ty1, ty2], dim=-1), dim=-1)[0]
    tymax = torch.max(torch.stack([ty1, ty2], dim=-1), dim=-1)[0]
    tmin = torch.max(torch.stack([tmin, tymin], dim=-1), dim=-1)[0]
    tmax = torch.min(torch.stack([tmax, tymax], dim=-1), dim=-1)[0]
    hit_local = tmin.unsqueeze(-1) * d_local + o_local
    hit_world = rotate(hit_local, rot.unsqueeze(-1)) + c
    collision = (tmax >= tmin) & (tmin > 0.0)
    dist = torch.linalg.norm(o - hit_world, dim=-1)
    return torch.where(collision, dist, torch.full_like(dist, max_range))


def _rays_to_line(center, line_rot, length, origin, angles, max_range):
    """Ray / segment intersection (ref core.py:1544-1626); ``line_rot [B,1]``."""
    B, R = angles.shape
    o = origin.unsqueeze(1).expand(B, R, 2)
    c = center.unsqueeze(1).expand(B, R, 2)
    rot = line_rot.expand(B, R)
    L = torch.tensor(length, dtype=torch.float32)
    r = torch.stack([torch.cos(rot), torch.sin(rot)], dim=-1) * L
    s = torch.stack([torch.cos(angles), torch.sin(angles)], dim=-1)
    rxs = G.cross2(r, s)
    t = G.cross2(o - c, s / rxs)
    u = G.cross2(o - c, r / rxs)
    d = torch.linalg.norm(u * s, dim=-1)
    miss = (rxs == 0.0) | (t > 0.5) | (t < -0.5) | (u < 0.0)
    return torch.where(miss.squeeze(-1), torch.full_like(d, max_range), d)


def cast_rays(tables: P.PlanTables, pos, rot, src: int, targets: List[int], angles, max_range: float):
    """Minimum range over ``targets`` for rays leaving entity ``src`` at ``angles [B,R]``.

    The reference takes the minimum over boxes, then spheres, then lines (core.py:1693-1786);
    a minimum is order-independent so targets are simply visited in entity order.
    """
    desc = tables.desc
    origin = pos[:, src]
    best = torch.full_like(angles, max_range)
    for t in targets:
        e = desc.entities[t]
        if e["shape"] == P.SHAPE_SPHERE:
            d = _rays_to_sphere(pos[:, t], e["d0"], origin, angles, max_range)
        elif e["shape"] == P.SHAPE_BOX:
            d = _rays_to_box(pos[:, t], rot[:, t : t + 1], e["d0"], e["d1"], origin, angles, max_range)
        else:
            d = _rays_to_line(pos[:, t], rot[:, t : t + 1], e["d0"], origin, angles, max_range)
        best = torch.min(torch.stack([best, d], dim=-1), dim=-1)[0]
    return best


# --------------------------------------------------------------------------------------
# distance / overlap queries
# --------------------------------------------------------------------------------------
def distance_from_point(tables: P.PlanTables, pos, rot, ent: int, point):
    """ref core.py:1788-1820."""
    e = tables.desc.entities[ent]
    p, r = pos[:, ent], rot[:, ent : ent + 1]
    if e["shape"] == P.SHAPE_SPHERE:
        return torch.linalg.vector_norm(p - point, dim=-1) - e["d0"]
    if e["shape"] == P.SHAPE_BOX:
        cp = G.closest_point_box(p, r, e["d0"], e["d1"], point)
    else:
        cp = G.closest_point_line(p, r, e["d0"], point)
    return torch.linalg.vector_norm(point - cp, dim=-1) - LINE_MIN_DIST


def _order(tables, a, b, first_shape, second_shape):
    ea = tables.desc.entities[a]
    return (a, b) if ea["shape"] == first_shape else (b, a)


def pair_overlap(tables: P.PlanTables, pos, rot, a: int, b: int):
    """ref core.py:1907-1969."""
    ents = tables.desc.entities
    shapes = {ents[a]["shape"], ents[b]["shape"]}
    if shapes == {P.SHAPE_BOX, P.SHAPE_SPHERE} and ents[a]["shape"] != ents[b]["shape"]:
        box, sph = _order(tables, a, b, P.SHAPE_BOX, P.SHAPE_SPHERE)
        eb = ents[box]
        pb, ps = pos[:, box], pos[:, sph]
        cp = G.closest_point_box(pb, rot[:, box : box + 1], eb["d0"], eb["d1"], ps)
        d_sphere_cp = torch.linalg.vector_norm(ps - cp, dim=-1)
        d_sphere_box = torch.linalg.vector_norm(ps - pb, dim=-1)
        d_cp_box = torch.linalg.vector_norm(pb - cp, dim=-1)
        dist_min = ents[sph]["d0"] + LINE_MIN_DIST
        return (d_sphere_box < d_cp_box) + (d_sphere_cp < dist_min)
    return pair_distance(tables, pos, rot, a, b) < 0


def pair_distance(tables: P.PlanTables, pos, rot, a: int, b: int):
    """ref core.py:1822-1905."""
    ents = tables.desc.entities
    sa, sb = ents[a]["shape"], ents[b]["shape"]
    if sa == P.SHAPE_SPHERE and sb == P.SHAPE_SPHERE:
        return distance_from_point(tables, pos, rot, a, pos[:, b]) - ents[b]["d0"]
    if {sa, sb} == {P.SHAPE_BOX, P.SHAPE_SPHERE}:
        box, sph = _order(tables, a, b, P.SHAPE_BOX, P.SHAPE_SPHERE)
        out = distance_from_point(tables, pos, rot, box, pos[:, sph]) - ents[sph]["d0"]
        return torch.where(pair_overlap(tables, pos, rot, a, b), torch.full_like(out, -1.0), out)
    if {sa, sb} == {P.SHAPE_LINE, P.SHAPE_SPHERE}:
        line, sph = _order(tables, a, b, P.SHAPE_LINE, P.SHAPE_SPHERE)
        return distance_from_point(tables, pos, rot, line, pos[:, sph]) - ents[sph]["d0"]
    ra, rb = rot[:, a : a + 1], rot[:, b : b + 1]
    if sa == P.SHAPE_LINE and sb == P.SHAPE_LINE:
        p1, p2 = G.closest_points_line_line(pos[:, a], ra, ents[a]["d0"], pos[:, b], rb, ents[b]["d0"])
    elif {sa, sb} == {P.SHAPE_BOX, P.SHAPE_LINE}:
        box, line = _order(tables, a, b, P.SHAPE_BOX, P.SHAPE_LINE)
        p1, p2 = G.closest_line_box(
            pos[:, box],
            rot[:, box : box + 1],
            ents[box]["d0"],
            ents[box]["d1"],
            pos[:, line],
            rot[:, line : line + 1],
            ents[line]["d0"],
        )
    else:
        p1, p2 = G.closest_box_box(
            pos[:, a], ra, ents[a]["d0"], ents[a]["d1"], pos[:, b], rb, ents[b]["d0"], ents[b]["d1"]
        )
    return torch.linalg.vector_norm(p1 - p2, dim=-1) - LINE_MIN_DIST
