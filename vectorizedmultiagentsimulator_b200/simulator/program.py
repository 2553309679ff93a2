"""Post-step programs: a scenario's reward / done glue as ONE kernel launch, fused with the observation gather.

The callbacks of a typical scenario (ref ``scenarios/balance.py:197-263``, ``transport.py:139-190``) are a
few ``is_overlapping`` / ``get_distance`` queries, the distance-shaping pattern and a handful of
elementwise operations on ``[B]`` tensors.  As torch ops each of them is a kernel of a few microseconds in
the step graph; as a :class:`StepProgram` they are a short instruction list one thread per env interprets
(``vmas_b200_post_step``), launched together with the observation gather of an
:class:`~.observe.ObservationPlan`.  On the CPU oracle backend the same program is interpreted with the
torch ops it replaces, so a scenario written on it behaves identically on both backends (and is checked
against the reference there).

    p = StepProgram(world)
    on_line, on_floor, on_goal = p.overlap(line, floor), p.overlap(package, floor), p.overlap(package, goal)
    on_ground = p.logical_or(on_line, on_floor)
    pos_rew, dist = p.shaping(package, goal, factor, prev=lambda: self.global_shaping)
    ground_rew = p.where(on_ground, p.const(-10.0), p.const(0.0))
    self.rew_out = p.store(p.add(ground_rew, pos_rew))
    self.done_out = p.store(p.logical_or(on_ground, on_goal), torch.bool)
    ...
    obs = p.run(observe=plan)          # one launch: outputs land in the ``.tensor`` of every store

Registers hold fp32 values (booleans are 0 / 1); at most 32 registers, 64 instructions, 16 buffers.
"""
from __future__ import annotations

from typing import Callable, List, Optional, Tuple, Union

import torch
from torch import Tensor

(
    OP_OVERLAP, OP_DISTANCE, OP_CENTER_DISTANCE, OP_SHAPING, OP_LOAD_F32, OP_LOAD_BOOL, OP_CONST, OP_ADD, OP_SUB, OP_MUL,
    OP_MIN, OP_MAX, OP_NEG, OP_OR, OP_AND, OP_NOT, OP_LT, OP_LE, OP_WHERE, OP_STORE_F32, OP_STORE_BOOL,
) = range(1, 22)
#: the env's step counter after this step's increment (operand ``a``: the counter's buffer slot).  A load of that
#: buffer but in the one-kernel step, which counts the step itself; only ``Environment`` splices it into a program
#: that step kernel runs (``_splice_limit``)
OP_STEP_COUNT = 22
MAX_INSTR, MAX_BUFFERS, MAX_REGS = 64, 16, 32

Buffer = Union[Tensor, Callable[[], Tensor]]


class Reg:
    """A per-env scalar of the program (fp32; ``is_bool``: a 0 / 1 flag)."""

    __slots__ = ("index", "is_bool")

    def __init__(self, index: int, is_bool: bool):
        self.index, self.is_bool = index, is_bool


class Output:
    """Where a ``store`` lands: ``.tensor`` is a ``[B]`` tensor that every ``run`` overwrites."""

    __slots__ = ("tensor", "dtype", "_slot")

    def __init__(self, dtype):
        self.tensor: Optional[Tensor] = None
        self.dtype = dtype
        self._slot = -1


class StepProgram:
    def __init__(self, world):
        self.world = world
        self.instr: List[Tuple] = []  # (op, dst, a, b, arg, imm, entities)
        self.buffers: List[Buffer] = []
        self.outputs: List[Output] = []
        self.n_regs = 0
        self._finalized = False
        self.device_cache = {}  # id(backend) -> (plan version, compiled struct)

    # -- building --------------------------------------------------------------------------
    def _reg(self, is_bool: bool, n: int = 1) -> Reg:
        assert not self._finalized, "the program is already finalized"
        r = Reg(self.n_regs, is_bool)
        self.n_regs += n
        assert self.n_regs <= MAX_REGS, f"a step program has at most {MAX_REGS} registers"
        return r

    def _emit(self, op, dst=0, a=0, b=0, arg=0, imm=0.0, entities=None):
        assert len(self.instr) < MAX_INSTR, f"a step program has at most {MAX_INSTR} instructions"
        self.instr.append((op, dst, a, b, arg, float(imm), entities))

    def _buffer(self, buf: Buffer) -> int:
        self.buffers.append(buf)
        assert len(self.buffers) <= MAX_BUFFERS, f"a step program has at most {MAX_BUFFERS} buffers"
        return len(self.buffers) - 1

    def overlap(self, a, b) -> Reg:
        """``world.is_overlapping(a, b)`` (ref core.py:1907-1969)."""
        r = self._reg(True)
        self._emit(OP_OVERLAP, r.index, entities=(a, b))
        return r

    def distance(self, a, b) -> Reg:
        """``world.get_distance(a, b)`` (ref core.py:1822-1905)."""
        r = self._reg(False)
        self._emit(OP_DISTANCE, r.index, entities=(a, b))
        return r

    def center_distance(self, a, b) -> Reg:
        """``|a.state.pos - b.state.pos|``."""
        r = self._reg(False)
        self._emit(OP_CENTER_DISTANCE, r.index, entities=(a, b))
        return r

    def shaping(self, a, b, factor: float, prev: Buffer) -> Tuple[Reg, Reg]:
        """The distance-shaping pattern: ``dist = |pos_a - pos_b|; rew = prev - dist * factor;
        prev <- dist * factor`` (``prev``: the carried ``[B]`` tensor, or a callable returning it).
        Returns ``(rew, dist)``."""
        rew = self._reg(False, 2)
        self._emit(OP_SHAPING, rew.index, a=self._buffer(prev), imm=factor, entities=(a, b))
        return rew, Reg(rew.index + 1, False)

    def load(self, buf: Buffer, is_bool: bool = False) -> Reg:
        r = self._reg(is_bool)
        self._emit(OP_LOAD_BOOL if is_bool else OP_LOAD_F32, r.index, a=self._buffer(buf))
        return r

    def const(self, value: float) -> Reg:
        r = self._reg(False)
        self._emit(OP_CONST, r.index, imm=value)
        return r

    def _binary(self, op, x: Reg, y: Reg, is_bool: bool) -> Reg:
        r = self._reg(is_bool)
        self._emit(op, r.index, x.index, y.index)
        return r

    def add(self, x, y): return self._binary(OP_ADD, x, y, False)  # noqa: E704
    def sub(self, x, y): return self._binary(OP_SUB, x, y, False)  # noqa: E704
    def mul(self, x, y): return self._binary(OP_MUL, x, y, False)  # noqa: E704
    def minimum(self, x, y): return self._binary(OP_MIN, x, y, False)  # noqa: E704
    def maximum(self, x, y): return self._binary(OP_MAX, x, y, False)  # noqa: E704
    def logical_or(self, x, y): return self._binary(OP_OR, x, y, True)  # noqa: E704
    def logical_and(self, x, y): return self._binary(OP_AND, x, y, True)  # noqa: E704
    def lt(self, x, y): return self._binary(OP_LT, x, y, True)  # noqa: E704
    def le(self, x, y): return self._binary(OP_LE, x, y, True)  # noqa: E704

    def neg(self, x: Reg) -> Reg:
        r = self._reg(False)
        self._emit(OP_NEG, r.index, x.index)
        return r

    def logical_not(self, x: Reg) -> Reg:
        r = self._reg(True)
        self._emit(OP_NOT, r.index, x.index)
        return r

    def where(self, cond: Reg, x: Reg, y: Reg) -> Reg:
        r = self._reg(x.is_bool and y.is_bool)
        self._emit(OP_WHERE, r.index, cond.index, x.index, arg=y.index)
        return r

    def store(self, x: Reg, dtype=None) -> Output:
        """Registers ``x`` as an output; its ``[B]`` tensor (fp32, or bool for flags) exists after
        :meth:`finalize` and is overwritten by every :meth:`run`."""
        dtype = dtype or (torch.bool if x.is_bool else torch.float32)
        assert dtype in (torch.float32, torch.bool)
        out = Output(dtype)
        out._slot = len(self.buffers)
        self.buffers.append(out)
        assert len(self.buffers) <= MAX_BUFFERS, f"a step program has at most {MAX_BUFFERS} buffers"
        self._emit(OP_STORE_BOOL if dtype == torch.bool else OP_STORE_F32, 0, x.index, out._slot)
        self.outputs.append(out)
        return out

    def finalize(self) -> "StepProgram":
        """Allocates the outputs: one contiguous fp32 block and one bool block, rows in store order (so
        a CUDA-graph step hands each block out with one copy)."""
        if self._finalized:
            return self
        B, dev = self.world.batch_dim, self.world.device
        floats = [o for o in self.outputs if o.dtype == torch.float32]
        bools = [o for o in self.outputs if o.dtype == torch.bool]
        if floats:
            pool = torch.zeros(len(floats), B, dtype=torch.float32, device=dev)
            for i, o in enumerate(floats):
                o.tensor = pool[i]
        if bools:
            pool = torch.zeros(len(bools), B, dtype=torch.bool, device=dev)
            for i, o in enumerate(bools):
                o.tensor = pool[i]
        self._finalized = True
        return self

    def instructions(self, index_of) -> List[Tuple]:
        """``[(op, dst, a, b, arg, imm)]`` with the entities of query instructions resolved to slab indices
        (``arg = index_a | index_b << 16``), as ``VmasProgInstr`` holds them."""
        out = []
        for op, dst, a, b, arg, imm, entities in self.instr:
            if entities is not None:
                arg = index_of(entities[0]) | (index_of(entities[1]) << 16)
            out.append((op, dst, a, b, arg, imm))
        return out

    # -- running ---------------------------------------------------------------------------
    def resolve(self, buf) -> Tensor:
        if isinstance(buf, Output):
            return buf.tensor
        return buf() if callable(buf) else buf

    def run(self, observe=None) -> Optional[Tensor]:
        """Executes the program for every env (one launch on CUDA, fused with the observation gather of
        ``observe``, an ``ObservationPlan``).  Returns the ``[rows, B, width]`` observation block, or None."""
        self.finalize()
        return self.world._get_backend().run_program(self, observe)
