"""Observation blocks: every agent's observation assembled on the device in one or two launches.

The reference builds an observation per agent from slices and ``torch.cat``
(``vmas/scenarios/balance.py:236-262``, ``navigation.py:252-265``,
``flocking.py:186-199``): a dozen tiny kernels per agent per step.  Here a scenario describes its
observation once as rows of *terms*; the world compiles the rows into a column table and
``World.observe(plan)`` fills the whole ``[rows, batch_dim, width]`` block with
``vmas_b200_gather_observations`` (state-slab terms) and ``vmas_b200_cast_rays_batched`` (LIDAR
terms, written straight into their columns).  Row ``i`` of the block is a contiguous
``[batch_dim, width]`` tensor — the layout ``Environment.step`` hands out per agent.

Arithmetic is what the per-term torch expressions compute (fp32 subtraction, ``torch.remainder``),
so the block is bit-identical to the ``torch.cat`` formulation.
"""
from __future__ import annotations

import struct
from typing import List, Optional, Sequence

import numpy as np

OP_SKIP, OP_COPY, OP_DIFF, OP_REMAINDER, OP_BUFFER, OP_REG = 0, 1, 2, 3, 4, 5
MAX_BUFFERS = 8
FIELD_POS, FIELD_VEL, FIELD_ROT, FIELD_ANG_VEL = 0, 1, 2, 3
_FIELDS = {"pos": (FIELD_POS, 2), "vel": (FIELD_VEL, 2), "rot": (FIELD_ROT, 1), "ang_vel": (FIELD_ANG_VEL, 1)}


class Term:
    """One group of adjacent observation columns."""

    width = 0


class _State(Term):
    def __init__(self, field: str, entity, minus=None, modulus: Optional[float] = None):
        self.field, self.entity, self.minus, self.modulus = field, entity, minus, modulus
        self.width = _FIELDS[field][1]


class _Lidar(Term):
    def __init__(self, sensor, range_minus_distance: bool):
        self.sensor, self.range_minus_distance = sensor, range_minus_distance
        self.width = int(sensor._angles.shape[1])


class _Blank(Term):
    def __init__(self, width: int):
        self.width = int(width)


def pos(entity) -> Term:
    return _State("pos", entity)


def vel(entity) -> Term:
    return _State("vel", entity)


def rot(entity) -> Term:
    return _State("rot", entity)


def ang_vel(entity) -> Term:
    return _State("ang_vel", entity)


def rel_pos(a, b) -> Term:
    """``a.state.pos - b.state.pos``"""
    return _State("pos", a, minus=b)


def rel_vel(a, b) -> Term:
    """``a.state.vel - b.state.vel``"""
    return _State("vel", a, minus=b)


def rot_remainder(entity, modulus: float) -> Term:
    """``entity.state.rot % modulus``"""
    return _State("rot", entity, modulus=float(modulus))


class _Buffer(Term):
    width = 1

    def __init__(self, source):
        self.source = source


def value(source) -> Term:
    """One column holding a per-env fp32 value another producer computed: ``source`` is a ``[B]`` fp32 tensor, a
    callable returning one, or a ``program.Output`` (fp32) — e.g. a flag of the scenario's step program that is
    also part of the observation (ref scenarios/transport.py:177-183, ``package.on_goal``).  Read when the block
    is assembled: the producer must have run before ``World.observe`` / within the same ``StepProgram.run``."""
    return _Buffer(source)


def lidar(sensor, range_minus_distance: bool = False) -> Term:
    """The readings of ``sensor`` (``sensor.measure()``), or ``max_range - readings``."""
    return _Lidar(sensor, range_minus_distance)


def blank(width: int) -> Term:
    """Columns the scenario writes itself into the returned block (left untouched here)."""
    return _Blank(width)


def _f32_bits(x: float) -> int:
    return struct.unpack("<i", struct.pack("<f", float(np.float32(x))))[0]


class ObservationPlan:
    """Rows of terms, compiled against a world's entity order on first use."""

    def __init__(self, rows: Sequence[Sequence[Term]]):
        self.rows: List[List[Term]] = [list(r) for r in rows]
        widths = {sum(t.width for t in r) for r in self.rows}
        if len(widths) != 1:
            raise ValueError(f"every observation row must have the same width, got {sorted(widths)}")
        self.width = widths.pop()
        self.n_rows = len(self.rows)
        self._compiled = None  # (plan version, columns, lidars)
        self.buffer_sources = []
        self.device_cache = {}  # backend-owned device copies, keyed by the backend

    def column_of(self, row: int, term: Term) -> int:
        c = 0
        for t in self.rows[row]:
            if t is term:
                return c
            c += t.width
        raise KeyError("term is not part of this row")

    def compile(self, world):
        """``(columns int32 [rows, width, 4], lidars)`` with
        ``lidars = [(row, first column, sensor, range_minus_distance)]``."""
        version = world._plan_version
        if self._compiled is not None and self._compiled[0] == version:
            return self._compiled[1], self._compiled[2]
        index = {id(e): i for i, e in enumerate(world.entities)}
        cols = np.zeros((self.n_rows, self.width, 4), dtype=np.int32)
        lidars = []
        self.buffer_sources = []  # what OP_BUFFER columns read, in the order of their indices
        for r, row in enumerate(self.rows):
            c = 0
            for t in row:
                if isinstance(t, _State):
                    field, comps = _FIELDS[t.field]
                    for k in range(comps):
                        src = (field << 24) | (comps * index[id(t.entity)] + k)
                        if t.minus is not None:
                            cols[r, c + k] = (OP_DIFF, src, (field << 24) | (comps * index[id(t.minus)] + k), 0)
                        elif t.modulus is not None:
                            cols[r, c + k] = (OP_REMAINDER, src, 0, _f32_bits(t.modulus))
                        else:
                            cols[r, c + k] = (OP_COPY, src, 0, 0)
                elif isinstance(t, _Lidar):
                    lidars.append((r, c, t.sensor, t.range_minus_distance))
                elif isinstance(t, _Buffer):
                    known = [k for k, src in enumerate(self.buffer_sources) if src is t.source]
                    if not known:
                        if len(self.buffer_sources) >= MAX_BUFFERS:
                            raise ValueError(f"an observation plan reads at most {MAX_BUFFERS} value buffers")
                        self.buffer_sources.append(t.source)
                        known = [len(self.buffer_sources) - 1]
                    cols[r, c] = (OP_BUFFER, known[0], 0, 0)
                c += t.width
        flips = {f for _, _, _, f in lidars}
        if len(flips) > 1:
            raise ValueError("all LIDAR terms of one plan must use the same range_minus_distance setting")
        self._compiled = (version, cols, lidars)
        self.device_cache.clear()
        return cols, lidars

    def resolve_buffers(self):
        """The ``[B]`` fp32 tensors the plan's value columns read, in column-index order."""
        out = []
        for src in self.buffer_sources:
            t = src.tensor if hasattr(src, "tensor") and hasattr(src, "_slot") else (src() if callable(src) else src)
            out.append(t)
        return out
