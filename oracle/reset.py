"""ORACLE (test infrastructure, not product code) — episode reset on the CPU, in numpy.

Restates the reference's respawn procedure
(``vmas/simulator/utils.py:241-319`` ``ScenarioUtils.spawn_entities_randomly`` /
``find_random_pos_for_entity``: per entity, propose a uniform position in the bounds and re-draw it
in the envs where it is closer than ``min_dist`` to an occupied position) and the state zeroing of
``World.reset`` (``core.py:1179-1181`` → ``EntityState._reset`` ``core.py:286-296``), with the
counter-based random stream the CUDA kernels use (``csrc/reset.cuh``), so the kernels can be checked
bit for bit.

What is pinned and what is not.  The *procedure* (sequential placement, rejection against the
occupied set, uniform proposals in the bounds, first accepted proposal wins per env) follows the
reference and is checked against it statistically (``tests/test_reset_oracle.py`` compares the
distributions of the reference's own sampler and of this one).  The random *stream* cannot be
pinned to the reference: the reference draws from torch's global generator, whose sequence differs
between devices (CPU: mt19937, CUDA: Philox with torch's own offset bookkeeping), so there is no
seed-for-seed equality to preserve on a GPU — the reference itself does not have it.  The generator
here is Philox4x32-10 (Salmon, Moraes, Dror, Shaw: "Parallel random numbers: as easy as 1, 2, 3",
SC'11), checked against the published known-answer vectors of Random123.
"""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np

_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = np.uint32(0x9E3779B9), np.uint32(0xBB67AE85)
_LOW = np.uint64(0xFFFFFFFF)
_SHIFT = np.uint64(32)


def philox4x32_10(counter, key):
    """Philox4x32 with 10 rounds.  ``counter``: 4 uint32 arrays (broadcastable), ``key``: 2 uint32."""
    c0, c1, c2, c3 = (np.asarray(c, dtype=np.uint32) for c in counter)
    c0, c1, c2, c3 = np.broadcast_arrays(c0, c1, c2, c3)
    k0, k1 = np.uint32(key[0]), np.uint32(key[1])
    with np.errstate(over="ignore"):
        for _ in range(10):
            p0 = _M0 * c0.astype(np.uint64)
            p1 = _M1 * c2.astype(np.uint64)
            n0 = (p1 >> _SHIFT).astype(np.uint32) ^ c1 ^ k0
            n2 = (p0 >> _SHIFT).astype(np.uint32) ^ c3 ^ k1
            c1 = (p1 & _LOW).astype(np.uint32)
            c3 = (p0 & _LOW).astype(np.uint32)
            c0, c2 = n0, n2
            k0 = np.uint32((int(k0) + int(_W0)) & 0xFFFFFFFF)
            k1 = np.uint32((int(k1) + int(_W1)) & 0xFFFFFFFF)
    return c0, c1, c2, c3


def _uniform(bits, lo: np.float32, span: np.float32):
    """24 random bits → ``lo + u * span`` with ``u`` in [0, 1), every operation rounded to fp32."""
    u = (bits >> np.uint32(8)).astype(np.float32) * np.float32(2.0**-24)
    return (lo + (u * span).astype(np.float32)).astype(np.float32)


def _too_close(p, q, min_dist: np.float32):
    """``|p - q| < min_dist`` in fp32: sqrt(dx*dx + dy*dy), each operation rounded on its own."""
    dx = (p[..., 0] - q[..., 0]).astype(np.float32)
    dy = (p[..., 1] - q[..., 1]).astype(np.float32)
    return np.sqrt(((dx * dx).astype(np.float32) + (dy * dy).astype(np.float32)).astype(np.float32)) < min_dist


def selected_envs(batch_dim: int, env_index: Optional[int], env_mask) -> np.ndarray:
    """Indices of the envs a reset call touches (int → that env, mask → flagged envs, neither → all)."""
    if env_index is not None and env_index >= 0:
        return np.array([env_index], dtype=np.int64)
    if env_mask is None:
        return np.arange(batch_dim, dtype=np.int64)
    return np.nonzero(np.asarray(env_mask).astype(bool))[0].astype(np.int64)


def reset_state(state: dict, reset_count: Optional[np.ndarray], env_index=None, env_mask=None) -> None:
    """``World.reset(env_index)``: zero every state tensor (``[B, ...]`` numpy arrays, in place) in the
    selected envs and bump their episode counters."""
    some = next(iter(state.values()))
    envs = selected_envs(some.shape[0], env_index, env_mask)
    for arr in state.values():
        arr[envs] = 0.0
    if reset_count is not None:
        reset_count[envs] += 1


def spawn_entities(
    pos: np.ndarray,
    entities: Sequence[int],
    *,
    min_dist: float,
    x_bounds,
    y_bounds,
    seed: int,
    stream_id: int = 0,
    reset_count: Optional[np.ndarray] = None,
    occupied_entities: Sequence[int] = (),
    occupied: Optional[np.ndarray] = None,
    env_index: Optional[int] = None,
    env_mask=None,
    max_tries: int = 1 << 16,
    env_offset: int = 0,
):
    """Places ``len(entities)`` positions per selected env; ``pos`` (fp32 ``[B, E, 2]``) is updated
    in place for entries ``>= 0`` of ``entities``.

    Returns ``(out, exhausted)``: ``out`` fp32 ``[B, n_spawn, 2]`` holds the drawn positions in the
    rows of the selected envs (zeros elsewhere), ``exhausted`` counts the envs in which some draw hit
    ``max_tries``.  ``occupied``: fp32 ``[B, K, 2]`` or ``[1, K, 2]`` (shared by all envs).
    ``env_offset``: index of env 0 in the whole job when ``pos`` is one shard of it.
    """
    assert pos.dtype == np.float32 and pos.ndim == 3 and pos.shape[2] == 2
    assert 0 < len(entities) <= 64 and 0 < max_tries <= 1 << 27
    B = pos.shape[0]
    envs = selected_envs(B, env_index, env_mask)
    n_spawn = len(entities)
    out = np.zeros((B, n_spawn, 2), dtype=np.float32)
    if envs.size == 0:
        return out, 0
    key = (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    episode = (reset_count[envs] if reset_count is not None else np.zeros(envs.size)).astype(np.uint32)
    x_lo, y_lo = np.float32(x_bounds[0]), np.float32(y_bounds[0])
    span_x = np.float32(np.float32(x_bounds[1]) - x_lo)
    span_y = np.float32(np.float32(y_bounds[1]) - y_lo)
    md = np.float32(min_dist)
    extra = None
    if occupied is not None and occupied.shape[1] > 0:
        occupied = np.asarray(occupied, dtype=np.float32)
        assert occupied.shape[0] in (1, B), "occupied must be [B, K, 2] or [1, K, 2]"
        if occupied.shape[0] == B:
            extra = occupied[envs]
        else:  # the same points for every env
            extra = np.broadcast_to(occupied[0], (envs.size,) + occupied.shape[1:])
    global_env = ((envs + env_offset) & 0xFFFFFFFF).astype(np.uint32)  # the env's index in the whole (sharded) job
    exhausted = np.zeros(envs.size, dtype=bool)
    placed = np.zeros((envs.size, n_spawn, 2), dtype=np.float32)
    for i in range(n_spawn):
        slot = i << 26  # n_spawn <= 64, max_tries <= 2**27
        pending = np.ones(envs.size, dtype=bool)
        cur = np.zeros((envs.size, 2), dtype=np.float32)
        tries = 0
        r = None
        while pending.any():
            if tries % 2 == 0:
                r = philox4x32_10(
                    (global_env, episode, np.uint32(stream_id & 0xFFFFFFFF), np.uint32(slot | (tries // 2))), key
                )
            bx, by = (r[2], r[3]) if tries % 2 else (r[0], r[1])
            prop = np.stack([_uniform(bx, x_lo, span_x), _uniform(by, y_lo, span_y)], axis=-1)
            cur[pending] = prop[pending]
            bad = np.zeros(envs.size, dtype=bool)
            for j in occupied_entities:
                bad |= _too_close(cur, pos[envs, j], md)
            if extra is not None:
                for j in range(extra.shape[1]):
                    bad |= _too_close(cur, extra[:, j], md)
            for j in range(i):
                bad |= _too_close(cur, placed[:, j], md)
            pending &= bad
            tries += 1
            if tries >= max_tries:
                exhausted |= pending
                break
        placed[:, i] = cur
        if entities[i] >= 0:
            pos[envs, entities[i]] = cur
    out[envs] = placed
    return out, int(exhausted.sum())
