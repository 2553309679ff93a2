"""``Environment``: the vectorised env users step (ref vmas/simulator/environment/environment.py).

Same public surface and return layout as the reference (``step`` → ``obs, rews, dones, infos``
with one ``[num_envs, ...]`` tensor per policy agent).  What differs is underneath:

* ``world.step()`` is the CUDA physics kernel, not python;
* action validation can be *deferred* (``action_checks="deferred"``): the nan / range tests
  are evaluated on the device into a flag that is read back asynchronously and raised on the
  next call, instead of forcing two host syncs per agent per step (ref environment.py:621,
  651-653).  ``"sync"`` reproduces the reference timing of the asserts, ``"off"`` skips them;
* ``grad_enabled=True`` is rejected: the kernels are forward-only;
* ``auto_reset=True`` (extension) resets every env a step finishes inside that step, on the device:
  ``rewards / dones / infos`` describe the step that ended the episode, ``obs`` of a finished env is
  the first observation of its next episode — what ``obs = env.reset_at(dones)`` after the step
  would return, without the host in the loop (and, in graph mode, inside the captured graph);
* ``obs_dtype=torch.float16 | torch.bfloat16`` (extension) hands observations out as 16-bit values: every fp32
  leaf of every observation is exactly ``leaf.to(obs_dtype)`` of the fp32 one, rounded where the step already
  writes or copies its results (no launch of its own); the scenario still computes in fp32;
* ``cuda_graph=True`` captures one whole ``step`` (action decoding → dynamics → physics kernels →
  scenario reward / observation / done / info) into a CUDA graph after two eager warm-up steps
  and replays it afterwards: no Python, no per-kernel launch latency.  It requires a
  *graph-safe* scenario: no host synchronisation inside the step callbacks and every tensor that
  carries information from one step to the next updated in place (``BaseScenario.keep``).  The
  scenarios shipped with this package are; arbitrary third-party scenario files may not be,
  which is why the mode is opt-in.
"""
from __future__ import annotations

import contextlib
import ctypes
import math
import os
import random
from typing import Dict, List, Optional, Sequence, Union

import numpy as np
import torch
from torch import Tensor

from ..core import Agent, TorchVectorizedObject
from ..scenario import BaseScenario
from ..utils import AGENT_OBS_TYPE, DEVICE_TYPING, TorchUtils
from . import spaces

#: a captured step runs through ONE call into the library (``vmas_b200_env_step``: ingest, graph launch, hand-out)
_ONE_CALL_STEP = os.environ.get("VMAS_B200_ONE_CALL_STEP", "1") != "0"
#: ... which issues the step's launches itself when the captured graph holds nothing but library launches
_DIRECT_STEP = os.environ.get("VMAS_B200_DIRECT_STEP", "1") != "0"
#: ... as ONE whole-step kernel (substeps + the scenario's step program + observation rows) compiled for the
#: (world, program, plan) at hand; the capture waits this long for the compiler before going on without it
_WHOLE_STEP_KERNEL = os.environ.get("VMAS_B200_WHOLE_STEP_KERNEL", "1") != "0"
#: ... and writes the step's results straight into the fresh output blocks (no hand-out copy)
_WRITE_RESULTS_IN_PLACE = os.environ.get("VMAS_B200_RESULTS_IN_PLACE", "1") != "0"
#: ... with the action ingest and the broad phase inside that kernel too (holonomic agents; continuous, discrete or
#: multi-discrete actions)
_INGEST_IN_KERNEL = os.environ.get("VMAS_B200_INGEST_IN_KERNEL", "1") != "0"
_WHOLE_STEP_KERNEL_WAIT_S = float(os.environ.get("VMAS_B200_WHOLE_STEP_KERNEL_WAIT_S", "60"))


def _rebuild_outputs(node, fresh):
    """Output structure of a captured step with fresh leaves.  A module-level function: a
    recursive closure would form a reference cycle that keeps every step's output tensors alive
    until the cyclic garbage collector runs."""
    kind, payload = node
    if kind == "leaf":
        return fresh[payload]
    if kind == "dict":
        return {k: _rebuild_outputs(v, fresh) for k, v in payload.items()}
    if kind == "list":
        return [_rebuild_outputs(v, fresh) for v in payload]
    if kind == "tuple":
        return tuple(_rebuild_outputs(v, fresh) for v in payload)
    return payload


def splice_program(instrs, n_regs, n_slots, extra, feed_slot=None, feed_reg=None, count_slot=None):
    """One step program out of ``instrs`` (``[(op, dst, a, b, arg, imm)]`` over ``n_regs`` registers and ``n_slots``
    buffer slots) and ``extra`` behind it: ``extra``'s registers and buffer slots are numbered on from the first
    program's; its load of slot ``feed_slot`` (a result of the first program) is dropped and its readers read register
    ``feed_reg`` instead; its load of slot ``count_slot`` (the step counter) becomes ``OP_STEP_COUNT``.  ``extra`` may
    use loads, constants, the elementwise ops and stores.  Returns ``(instructions, registers, {extra's slot: slot})``."""
    from .. import program as SP

    regs, slots, fresh = {}, {}, []

    def reg(r):
        return regs[r]

    def slot(j):
        return slots.setdefault(j, n_slots + len(slots))

    def new_reg(r):
        regs[r] = n_regs + len(fresh)
        fresh.append(r)
        return regs[r]

    out = list(instrs)
    for op, dst, a, b, arg, imm in extra:
        if op in (SP.OP_LOAD_F32, SP.OP_LOAD_BOOL):
            if a == feed_slot:
                regs[dst] = feed_reg
                continue
            kind = SP.OP_STEP_COUNT if a == count_slot and op == SP.OP_LOAD_F32 else op
            out.append((kind, new_reg(dst), slot(a), 0, 0, 0.0))
        elif op == SP.OP_CONST:
            out.append((op, new_reg(dst), 0, 0, 0, imm))
        elif op in (SP.OP_NEG, SP.OP_NOT):
            out.append((op, new_reg(dst), reg(a), 0, 0, 0.0))
        elif op == SP.OP_WHERE:
            out.append((op, new_reg(dst), reg(a), reg(b), reg(arg), 0.0))
        elif SP.OP_ADD <= op <= SP.OP_LE:
            out.append((op, new_reg(dst), reg(a), reg(b), 0, 0.0))
        elif op in (SP.OP_STORE_F32, SP.OP_STORE_BOOL):
            out.append((op, 0, reg(a), slot(b), 0, 0.0))
        else:
            raise ValueError(f"op {op} cannot be spliced")
    return out, n_regs + len(fresh), slots


@contextlib.contextmanager
def local_seed(vmas_random_state):
    """Runs the body on the environment's private (torch-CPU, numpy, python) RNG streams."""
    outer = (torch.random.get_rng_state(), np.random.get_state(), random.getstate())
    torch.random.set_rng_state(vmas_random_state[0])
    np.random.set_state(vmas_random_state[1])
    random.setstate(vmas_random_state[2])
    try:
        yield
    finally:
        vmas_random_state[0] = torch.random.get_rng_state()
        vmas_random_state[1] = np.random.get_state()
        vmas_random_state[2] = random.getstate()
        torch.random.set_rng_state(outer[0])
        np.random.set_state(outer[1])
        random.setstate(outer[2])


def _seeded(method):
    def wrapper(self, *args, **kwargs):
        with local_seed(Environment.vmas_random_state):
            return method(self, *args, **kwargs)

    wrapper.__name__ = method.__name__
    wrapper.__doc__ = method.__doc__
    return wrapper


# opt-in (VMAS_B200_FORK_OBS=1): measured slower on balance / navigation / flocking at the BASELINE batch sizes
# on a B200 — the branches of the captured graph do not start together; on an H100 it is faster on navigation
# (DESIGN §7.3, §10)
_FORK_OBSERVATIONS = os.environ.get("VMAS_B200_FORK_OBS", "0") == "1"


#: what ``Environment(obs_dtype=...)`` accepts
OBS_DTYPES = (torch.float32, torch.float16, torch.bfloat16)


def check_obs_dtype(obs_dtype):
    if obs_dtype not in OBS_DTYPES:
        raise ValueError(f"obs_dtype must be torch.float32, torch.float16 or torch.bfloat16, not {obs_dtype!r}")


def _to_obs_dtype(x, dtype):
    """A fresh copy of one agent's observation with every fp32 leaf as ``dtype`` (other leaves cloned as they are)."""
    if isinstance(x, Tensor):
        return x.to(dtype) if x.dtype == torch.float32 else x.clone()
    return {k: _to_obs_dtype(v, dtype) for k, v in x.items()}


def _leaves(x):
    if isinstance(x, Tensor):
        yield x
    elif isinstance(x, dict):
        for v in x.values():
            yield from _leaves(v)
    elif isinstance(x, (list, tuple)):
        for v in x:
            yield from _leaves(v)


class Environment(TorchVectorizedObject):
    metadata = {"render.modes": ["human", "rgb_array"], "runtime.vectorized": True}
    vmas_random_state = [torch.random.get_rng_state(), np.random.get_state(), random.getstate()]

    def __init__(
        self,
        scenario: BaseScenario,
        num_envs: int = 32,
        device: DEVICE_TYPING = "cpu",
        max_steps: Optional[int] = None,
        continuous_actions: bool = True,
        seed: Optional[int] = None,
        dict_spaces: bool = False,
        multidiscrete_actions: bool = False,
        clamp_actions: bool = False,
        grad_enabled: bool = False,
        terminated_truncated: bool = False,
        action_checks: Optional[str] = None,
        cuda_graph: bool = False,
        auto_reset: bool = False,
        obs_dtype: torch.dtype = torch.float32,
        **kwargs,
    ):
        check_obs_dtype(obs_dtype)
        if multidiscrete_actions:
            assert (
                not continuous_actions
            ), "When asking for multidiscrete_actions, make sure continuous_actions=False"
        if grad_enabled:
            raise NotImplementedError(
                "grad_enabled=True is not supported: the CUDA physics kernels are forward-only"
            )
        with local_seed(Environment.vmas_random_state):
            self.scenario = scenario
            self.num_envs = num_envs
            TorchVectorizedObject.__init__(self, num_envs, torch.device(device))
            self.world = self.scenario.env_make_world(self.num_envs, self.device, **kwargs)

            self.agents = self.world.policy_agents
            self.n_agents = len(self.agents)
            self.max_steps = max_steps
            self.continuous_actions = continuous_actions
            self.dict_spaces = dict_spaces
            self.clamp_action = clamp_actions
            self.grad_enabled = grad_enabled
            self.terminated_truncated = terminated_truncated
            if action_checks is None:
                action_checks = "deferred" if self.device.type == "cuda" else "sync"
            assert action_checks in ("sync", "deferred", "off")
            self.action_checks = action_checks
            self._bad_action_flag = None  # device uint8 [1], set by deferred checks
            self._bad_action_host = None
            self._bad_action_event = None
            self._bad_action_messages = []
            if cuda_graph and self.device.type != "cuda":
                raise ValueError("cuda_graph=True needs a CUDA device")
            self.cuda_graph = cuda_graph
            self.auto_reset = auto_reset
            self.obs_dtype = obs_dtype
            if auto_reset and not self.scenario.supports_masked_reset:
                raise NotImplementedError(
                    f"auto_reset=True needs a scenario whose reset_world_at accepts a bool mask "
                    f"(supports_masked_reset); {type(self.scenario).__name__} takes an env index"
                )
            self._graph = None
            self._graph_inputs = None
            self._graph_outputs = None
            self._graph_plan_version = None
            self._graph_warmup_left = 2
            self._one_call = None
            self._one_call_state = "off"
            self.graph_replays = 0

            observations = self._reset(seed=seed)

            self.multidiscrete_actions = multidiscrete_actions
            self.action_space = self.get_action_space()
            self.observation_space = self.get_observation_space(observations)

            self.viewer = None
            self.headless = None
            self.visible_display = None
            self.text_lines = None

    # ------------------------------------------------------------------------------------
    # public API (each runs on the env's private RNG streams)
    # ------------------------------------------------------------------------------------
    @_seeded
    def reset(
        self,
        seed: Optional[int] = None,
        return_observations: bool = True,
        return_info: bool = False,
        return_dones: bool = False,
    ):
        """Resets all envs; returns observations for all envs and agents."""
        return self._reset(seed, return_observations, return_info, return_dones)

    @_seeded
    def reset_at(
        self,
        index: int,
        return_observations: bool = True,
        return_info: bool = False,
        return_dones: bool = False,
    ):
        """Resets env ``index``; returns observations for all agents (all envs).

        Extension of the reference API: ``index`` may be a ``[num_envs]`` bool tensor (e.g. the
        ``dones`` of the last step); every flagged env is reset in one pass on the device, without
        a host sync, where the reference needs one ``reset_at(i)`` per finished env.  Needs a
        scenario with ``supports_masked_reset``.
        """
        return self._reset_at(index, return_observations, return_info, return_dones)

    @_seeded
    def get_from_scenario(
        self,
        get_observations: bool,
        get_rewards: bool,
        get_infos: bool,
        get_dones: bool,
        dict_agent_names: Optional[bool] = None,
    ):
        return self._get_from_scenario(
            get_observations, get_rewards, get_infos, get_dones, dict_agent_names
        )

    @_seeded
    def seed(self, seed=None):
        return self._seed(seed)

    @_seeded
    def done(self):
        return self._done()

    def step(self, actions: Union[List, Dict]):
        """One vectorised step.

        Args:
            actions: list (or dict by agent name) with one ``[num_envs, action_size]`` tensor
                per policy agent.
        Returns:
            ``obs, rewards, dones, infos`` (or ``obs, rewards, terminated, truncated, infos``),
            lists (or dicts) with one entry per policy agent.
        """
        if self._graph is not None:
            # a graph replay runs no Python scenario code and draws no host random numbers:
            # the swap of the env's private RNG streams (3 get/set state pairs) is skipped
            return self._step(actions)
        with local_seed(Environment.vmas_random_state):
            return self._step(actions)

    # ------------------------------------------------------------------------------------
    def _reset(self, seed=None, return_observations=True, return_info=False, return_dones=False):
        if seed is not None:
            self._seed(seed)
        self.scenario.env_reset_world_at(env_index=None)
        if getattr(self, "steps", None) is not None:
            self.steps.zero_()  # in place: a captured step graph keeps reading this tensor
        else:
            self.steps = torch.zeros(self.num_envs, device=self.device)
        result = self._get_from_scenario(
            get_observations=return_observations,
            get_infos=return_info,
            get_rewards=False,
            get_dones=return_dones,
        )
        return result[0] if result and len(result) == 1 else result

    def _reset_at(self, index, return_observations=True, return_info=False, return_dones=False):
        if isinstance(index, Tensor):
            if index.dtype != torch.bool or index.shape != (self.num_envs,):
                raise ValueError("a tensor passed to reset_at must be a [num_envs] bool mask")
            if not self.scenario.supports_masked_reset:
                raise NotImplementedError(
                    f"{type(self.scenario).__name__}.reset_world_at takes an env index; resetting by mask "
                    "needs a scenario with supports_masked_reset = True"
                )
            index = index.to(self.device)
            self.scenario.env_reset_world_at(index)
            self.steps.masked_fill_(index, 0)
        else:
            self._check_batch_index(index)
            self.scenario.env_reset_world_at(index)
            self.steps[index] = 0
        result = self._get_from_scenario(
            get_observations=return_observations,
            get_infos=return_info,
            get_rewards=False,
            get_dones=return_dones,
        )
        return result[0] if result and len(result) == 1 else result

    def _get_from_scenario(
        self, get_observations, get_rewards, get_infos, get_dones, dict_agent_names=None, clone=True
    ):
        if not (get_infos or get_dones or get_rewards or get_observations):
            return
        by_name = self.dict_spaces if dict_agent_names is None else dict_agent_names
        # the reference clones everything it hands out (environment.py:278, 285, 294, 415);
        # graph mode clones once, outside the captured region, instead
        _c = (lambda t: t.clone()) if clone else (lambda t: t)
        _rc = TorchUtils.recursive_clone if clone else (lambda t: t)
        # observations: the same clone, or the conversion to 16 bits in its place (graph mode: the hand-out copy)
        _oc = _rc
        if clone and self.obs_dtype != torch.float32:
            _oc = lambda t: _to_obs_dtype(t, self.obs_dtype)  # noqa: E731

        def collect(fn):
            out = {} if by_name else []
            for agent in self.agents:
                value = fn(agent)
                if by_name:
                    out[agent.name] = value
                else:
                    out.append(value)
            return out

        # Experiment, off by default: a scenario whose observations read nothing but the world state (it
        # says so: ``observations_are_independent``) can have them computed on a side stream, next to the
        # reward / info / done callbacks instead of behind them (parallel branches of the captured graph).
        # Everything joins again before the results are handed out.
        fork = (
            get_observations
            and (get_rewards or get_infos or get_dones)
            and self.device.type == "cuda"
            and getattr(self.scenario, "observations_are_independent", False)
            and _FORK_OBSERVATIONS
        )
        obs = None
        if fork:
            main = torch.cuda.current_stream(self.device)
            if getattr(self, "_obs_stream", None) is None:
                self._obs_stream = torch.cuda.Stream(device=self.device)
            side = self._obs_stream
            side.wait_stream(main)
            with torch.cuda.stream(side):
                obs = collect(lambda a: _oc(self.scenario.observation(a)))
        # order matters: scenarios cache shared terms while computing agent 0's reward
        rewards = collect(lambda a: _c(self.scenario.reward(a))) if get_rewards else None
        if get_observations and not fork:
            obs = collect(lambda a: _oc(self.scenario.observation(a)))
        infos = collect(lambda a: _rc(self.scenario.info(a))) if get_infos else None
        if self.terminated_truncated:
            terminated = truncated = None
            if get_dones:
                terminated, truncated = self._done(clone)
            result = [obs, rewards, terminated, truncated, infos]
        else:
            dones = self._done(clone) if get_dones else None
            result = [obs, rewards, dones, infos]
        if fork:
            main.wait_stream(side)
            if not torch.cuda.is_current_stream_capturing():
                for leaf in _leaves(obs):  # allocated on the side stream, used by the caller on this one
                    leaf.record_stream(main)
        return [data for data in result if data is not None]

    def _seed(self, seed=None):
        if seed is None:
            seed = 0
        torch.manual_seed(seed)
        np.random.seed(seed)
        random.seed(seed)
        if getattr(self, "world", None) is not None:
            # the device-side respawn draws from a stream keyed by THIS env's seed, not by whatever
            # env seeded torch's global generator last (the random state is shared by all envs)
            self.world.spawn_seed = int(seed)
        if getattr(self, "auto_reset", False) and getattr(self, "_graph", None) is not None:
            # the captured step contains the respawn kernel, whose Philox key is the seed: capture again
            self._graph = None
            self._graph_warmup_left = 1
        return [seed]

    def _normalize_actions(self, actions) -> List[Tensor]:
        if isinstance(actions, Dict):
            by_name = actions
            actions = []
            for agent in self.agents:
                if agent.name not in by_name:
                    raise AssertionError(f"Agent '{agent.name}' not contained in action dict")
                actions.append(by_name[agent.name])
            assert (
                len(by_name) == self.n_agents
            ), f"Expecting actions for {self.n_agents}, got {len(by_name)} actions"
        assert (
            len(actions) == self.n_agents
        ), f"Expecting actions for {self.n_agents}, got {len(actions)} actions"
        actions = list(actions)
        sizes = self._action_sizes()
        n_env = self.num_envs
        if all(type(a) is Tensor and a.dim() == 2 and a.shape[0] == n_env and a.shape[1] == k for a, k in zip(actions, sizes)):
            return actions  # the common case: nothing to convert, nothing to report
        for i, agent in enumerate(self.agents):
            a = actions[i]
            if not isinstance(a, Tensor):
                a = torch.tensor(a, dtype=torch.float32, device=self.device)
            if a.dim() == 1:
                a = a.unsqueeze(-1)
            assert (
                a.shape[0] == self.num_envs
            ), f"Actions used in input of env must be of len {self.num_envs}, got {a.shape[0]}"
            expected = self.get_agent_action_size(agent)
            assert a.shape[1] == expected, (
                f"Action for agent {agent.name} has shape {a.shape[1]},"
                f" but should have shape {expected}"
            )
            actions[i] = a
        return actions

    def _action_sizes(self) -> List[int]:
        sizes = getattr(self, "_action_size_cache", None)
        if sizes is None or sizes[0] != self.world._plan_version or len(sizes[1]) != self.n_agents:
            sizes = self._action_size_cache = (
                self.world._plan_version,
                [self.get_agent_action_size(a) for a in self.agents],
            )
        return sizes[1]

    def _hold_host_actions(self, actions: List[Tensor]):
        """Pinned host action tensors are read by a kernel where they lie (no staging copy): they must not go
        back to torch's pinned-memory pool — and from there into another tensor — before that kernel has run.
        They are kept referenced until an event recorded behind the step has completed."""
        held = getattr(self, "_held_host_actions", None)
        if held is None:
            import collections

            held = self._held_host_actions = collections.deque()
        while held and held[0][0].query():
            held.popleft()
        if any(a.device.type == "cpu" for a in actions):
            event = torch.cuda.Event()
            event.record()
            held.append((event, list(actions)))

    def _step(self, actions):
        self._raise_deferred_action_errors()
        actions = self._normalize_actions(actions)
        if self.cuda_graph:
            result = self._step_graphed(actions)
        else:
            result = self._step_device(actions)
        if self.device.type == "cuda" and (
            getattr(self, "_held_host_actions", None) or any(a.device.type == "cpu" for a in actions)
        ):
            self._hold_host_actions(actions)
        self._launch_deferred_action_readback()
        return result

    def _fused_ingest_specs(self):
        """[(agent, dynamics code, u buffer)] if the fused action-ingest kernel reproduces what
        ``_set_action`` + ``env_process_action`` would do for every policy agent, else None.

        That holds for continuous, noise-free, non-communicating agents whose dynamics model the kernel
        implements (holonomic, holonomic with rotation, forward, rotation, static, differential drive,
        kinematic bicycle, drone) in scenarios that do not override ``process_action``.
        """
        version = self.world._plan_version
        cached = getattr(self, "_ingest_cache", None)
        if cached is not None and cached[0] == version:
            return cached[1]
        from ... import _native as N
        from ... import codegen

        specs = None
        ok = (
            self.device.type == "cuda"
            and self.action_checks != "sync"
            and type(self.scenario).process_action is BaseScenario.process_action
            and self.n_agents > 0
        )
        if ok:
            specs = []
            for agent in self.agents:
                noise = agent.action.u_noise
                noisy = (max(noise) if isinstance(noise, Sequence) else noise) > 0
                dyn = codegen.dynamics_code(agent.dynamics)  # exact types: a subclass may override process_action
                size_ok = 0 < agent.action_size <= 8 or (agent.action_size == 0 and dyn == N.DYN_NONE)
                if noisy or dyn is None or self._comm_dims(agent) > 0 or not size_ok:
                    specs = None
                    break
                u = torch.zeros(self.num_envs, agent.action_size, device=self.device, dtype=torch.float32)
                specs.append((agent, dyn, u))
        self._ingest_cache = (version, specs)
        return specs

    def _ingest_dtype(self):
        """What the fused ingest kernel reads: fp32 actions, or int64 indices in discrete spaces."""
        return torch.float32 if self.continuous_actions else torch.int64

    def _fused_ingest_applies(self, actions: List[Tensor]) -> bool:
        specs = self._fused_ingest_specs()
        if specs is None:
            return False
        if self.continuous_actions:
            # (an agent without action components — Static dynamics — hands in a [B, 0] tensor)
            # Pinned host tensors are read by the kernel where they lie (unified addressing: no staging copy, the
            # step's first kernel pulls the actions over PCIe itself); as with any asynchronous copy the caller
            # must leave them alone until the step has run.
            return all(
                a.dtype == torch.float32 and a.is_contiguous() and (a.device.type == "cuda" or a.is_pinned())
                for a in actions
            )
        # discrete spaces: int64 indices, [B, 1] (flat index of the product) or [B, action_size] (multi-discrete)
        return all(
            a.dtype == torch.int64 and a.is_contiguous() and a.device.type == "cuda" and a.dim() == 2
            and a.shape[1] == (s[0].action_size if self.multidiscrete_actions else 1)
            for a, s in zip(actions, specs)
        )

    def _apply_actions(self, actions: List[Tensor], fused: Optional[bool] = None, count_step: bool = True) -> bool:
        """Decodes the policy agents' actions into ``agent.action.u`` and slab forces.  Returns
        True if the fused kernel did it (scripted agents are then still to be processed).
        ``fused``: the caller's answer to ``_fused_ingest_applies(actions)``, if it already asked."""
        if self._fused_ingest_applies(actions) if fused is None else fused:
            specs = self._fused_ingest_specs()
            # one kernel instead of ~10 eager ops per agent (checks, scaling, force routing)
            flag = None
            if self.action_checks == "deferred":
                if self._bad_action_flag is None:
                    self._bad_action_flag = torch.zeros(1, dtype=torch.bool, device=self.device)
                    self._bad_action_messages = []
                flag = self._bad_action_flag
                msg = "an action is NaN or outside its agent's u_range"
                if msg not in self._bad_action_messages:
                    self._bad_action_messages.append(msg)
            # agents without action components (Static dynamics) have nothing to ingest
            live = [(a, s) for a, s in zip(actions, specs) if s[0].action_size > 0]
            N = self.world._get_backend()._native
            kind = (
                N.ACT_CONTINUOUS if self.continuous_actions
                else (N.ACT_MULTIDISCRETE if self.multidiscrete_actions else N.ACT_DISCRETE)
            )
            # the per-env step counter is incremented by the same launch (_finish_step then skips its add)
            counts = self.steps.dtype == torch.float32 and self.steps.is_contiguous() and bool(live)
            counter = self.steps if (counts and count_step) else None
            # ... and so does the broad phase of the coming step, if nothing can move an entity in between
            static_until_step = (
                type(self.scenario).pre_step is BaseScenario.pre_step and not self.world.scripted_agents and bool(live)
            )
            self.world._get_backend().ingest_actions(
                [a for a, _ in live], [s for _, s in live], self.clamp_action, flag, action_kind=kind, steps=counter,
                broad_phase=static_until_step,
            )
            self._steps_counted = counts  # (count_step=False: the caller's replay will count this step)
            for agent, _, u in specs:
                if agent.action._u is not u:  # the u buffers are static: bind them once
                    agent.action.u = u
            return True
        for action, agent in zip(actions, self.agents):
            self._set_action(action, agent)
        # scripted agents + scenario-specific processing + dynamics (action -> force/torque)
        for agent in self.world.agents:
            self.scenario.env_process_action(agent)
        return False

    def _finish_step(self, fused_ingest: bool, clone_outputs: bool = True):
        """Everything after the policy actions are decoded: scripted agents, physics, callbacks."""
        if fused_ingest:
            for agent in self.world.scripted_agents:
                self.scenario.env_process_action(agent)
        self.scenario.pre_step()
        self.world.step()
        self.scenario.post_step()
        if fused_ingest and getattr(self, "_steps_counted", False):
            self._steps_counted = False  # the ingest kernel already counted this step
        else:
            self.steps += 1
        if not self.auto_reset:
            backend = self.world._get_backend() if self.device.type == "cuda" else None
            if backend is not None:
                backend.step_programs = []  # (the programs whose outputs _done's step limit may read)
            try:
                return self._get_from_scenario(
                    get_observations=True, get_infos=True, get_rewards=True, get_dones=True, clone=clone_outputs
                )
            finally:
                if backend is not None:
                    backend.step_programs = None
        # auto-reset: rewards / infos / dones describe the step that just ran; every env it finished
        # is reset on the device (mask = dones, no host sync) and the observations are taken
        # afterwards, so a finished env hands out the first observation of its next episode.  The
        # first three are cloned before the reset touches anything they might alias.
        rest = self._get_from_scenario(
            get_observations=False, get_infos=True, get_rewards=True, get_dones=True, clone=True
        )
        finished = (rest[1] | rest[2]) if self.terminated_truncated else rest[1]
        self.scenario.env_reset_world_at(finished)
        self.steps.masked_fill_(finished, 0)
        obs = self._get_from_scenario(
            get_observations=True, get_infos=False, get_rewards=False, get_dones=False, clone=clone_outputs
        )
        return obs + rest

    def _step_device(self, actions: List[Tensor], clone_outputs: bool = True):
        """The device-side work of one step."""
        return self._finish_step(self._apply_actions(actions), clone_outputs)

    # ---- CUDA-graph mode -------------------------------------------------------------------
    def _step_graphed(self, actions: List[Tensor]):
        world = self.world
        if self._graph is not None and (
            self._graph_plan_version != world._plan_version
            or any(a.shape != s or a.dtype != d for a, (s, d) in zip(actions, self._graph_action_layout))
        ):
            self._graph = None  # the world or the action layout changed: capture again
            self._graph_warmup_left = 1
        if self._graph is None:
            if self._graph_warmup_left > 0:
                self._graph_warmup_left -= 1
                return self._step_device([a.to(self.device) for a in actions])
            self._capture(actions)
        if self._one_call_state == "on" and self._fused_ingest_applies(actions):
            return self._step_one_call(actions)
        if self._graph_inputs is None:
            # the fused ingest kernel reads the caller's tensors directly (one eager launch in
            # front of the replay; no staging copy into graph-owned input buffers)
            if not self._fused_ingest_applies(actions):
                # pinned host tensors are uploaded asynchronously (stream-ordered before the kernel)
                actions = [
                    a.to(self.device, self._ingest_dtype(), non_blocking=a.is_pinned() if a.device.type == "cpu" else False)
                    .contiguous()
                    for a in actions
                ]
            self._apply_actions(actions, fused=True)
        elif all(a.device == s.device and a.dtype == s.dtype for a, s in zip(actions, self._graph_inputs)):
            # one multi-tensor copy for all agents' actions
            torch._foreach_copy_(self._graph_inputs, list(actions))
        else:
            for static, a in zip(self._graph_inputs, actions):
                static.copy_(a, non_blocking=True)
        if self._one_call_state == "probe":
            # torch's replay advances the philox offset of a graph that draws random numbers; a raw
            # cudaGraphLaunch would replay the same numbers, so such a graph stays on torch's replay
            gen = torch.cuda.default_generators[self.device.index if self.device.index is not None else torch.cuda.current_device()]
            before = gen.get_offset()
            self._graph.replay()
            self._one_call_state = "on" if gen.get_offset() == before else "off"
        else:
            self._graph.replay()
        self.graph_replays += 1
        backend = world._get_backend()
        backend.launches += self._graph_launches
        backend._mask_ready = False  # (consumed by the substep kernel inside the replay)
        backend.after_step()  # periodic env re-ordering: eager launches between replays
        return self._unpack_graph_outputs()

    #: a run of adjacent output leaves at least this large is cloned straight from where the
    #: scenario wrote it instead of being gathered into the per-dtype buffer first
    PACK_ALONE_BYTES = 1 << 20

    def _pack_graph_outputs(self, outputs):
        """(inside the capture) lays the output leaves out as a few flat blocks — one per big contiguous
        run, one per dtype for the small leaves — and prepares the copy that hands them out.  With a 16-bit
        ``obs_dtype`` the fp32 observation leaves (``outputs[0]``) get blocks of that type to themselves,
        and the hand-out copy rounds them on the way."""
        N = self.world._get_backend()._native
        leaves = []

        def index(x):
            if isinstance(x, Tensor):
                leaves.append(x)
                return ("leaf", len(leaves) - 1)
            if isinstance(x, dict):
                return ("dict", {k: index(v) for k, v in x.items()})
            if isinstance(x, (list, tuple)):
                return ("list" if isinstance(x, list) else "tuple", [index(v) for v in x])
            return ("const", x)

        spec = index(outputs)
        index = None  # the recursive closure references itself: break the cycle
        n_obs = len(list(_leaves(outputs[0]))) if self.obs_dtype != torch.float32 else 0
        converted = [i < n_obs and t.dtype == torch.float32 for i, t in enumerate(leaves)]
        # Runs of leaves that already sit back to back in one allocation (e.g. the rows of a
        # batched [A, B, F] observation block) are handed out as ONE view.  A big run is its own
        # pack (cloned as is: no gather copy in the graph); the small rest is concatenated into
        # one flat buffer per dtype.
        runs = []  # [first leaf, n leaves, numel]
        for i, t in enumerate(leaves):
            if runs and t.is_contiguous() and t.numel() > 0:
                first, n, numel = runs[-1]
                head = leaves[first]
                if (
                    head.is_contiguous()
                    and head.dtype == t.dtype
                    and converted[first] == converted[i]
                    and t.untyped_storage().data_ptr() == head.untyped_storage().data_ptr()
                    and t.data_ptr() == head.data_ptr() + numel * head.element_size()
                ):
                    runs[-1] = [first, n + 1, numel + t.numel()]
                    continue
            runs.append([i, 1, t.numel()])
        packs = []  # (buffer the graph fills, leaf ids in order)
        small = {}
        for first, n, numel in runs:
            head = leaves[first]
            ids = list(range(first, first + n))
            if head.is_contiguous() and numel * head.element_size() >= self.PACK_ALONE_BYTES:
                packs.append((head.as_strided((numel,), (1,)), ids))
            else:
                small.setdefault((head.dtype, converted[first]), []).extend(ids)
        # The small leaves of a dtype form one output block too, but nothing gathers them inside the graph:
        # the hand-out copy reads every leaf where the scenario wrote it (sources[i] = the pieces of block
        # i, in order).  A non-contiguous leaf is made contiguous by a copy node (rare: scenarios return
        # fresh or [B]-row tensors).
        sources = [[pack] for pack, _ in packs]
        for _, ids in small.items():
            pieces = [leaves[i] if leaves[i].is_contiguous() else leaves[i].contiguous() for i in ids]
            total = sum(t.numel() for t in pieces)
            packs.append((None, ids))
            sources.append([t.reshape(-1) for t in pieces])
        # per block: what the hand-out copy makes of its fp32 sources (DTYPE_F32: a plain copy)
        kinds = [N.DTYPE_CODES[self.obs_dtype] if converted[ids[0]] else N.DTYPE_F32 for _, ids in packs]
        self._graph_out_blocks = [
            (sum(t.numel() for t in pieces), self.obs_dtype if kind else pieces[0].dtype)
            for pieces, kind in zip(sources, kinds)
        ]
        self._graph_out_block_kinds = kinds
        items, copies_per_block = [], []
        for block, pieces in enumerate(sources):
            offset = 0
            size = self._graph_out_blocks[block][1].itemsize
            for t in pieces:
                if t.numel():
                    items.append((t, block, offset))
                offset += t.numel() * size
        self._graph_out_copy = [
            N.CopyPlan(items[lo : lo + N.MAX_COPY_SEGMENTS], kinds) for lo in range(0, len(items), N.MAX_COPY_SEGMENTS)
        ]
        self._graph_out_spec = spec
        self._graph_out_shapes = [tuple(t.shape) for t in leaves]
        self._graph_out_packs = packs
        # per pack: runs of consecutive equal-shape leaves [(count, shape, numel per leaf)]
        layouts = []
        for _, ids in packs:
            layout = []
            for i in ids:
                shape = self._graph_out_shapes[i]
                if layout and layout[-1][1] == shape:
                    layout[-1][0] += 1
                else:
                    layout.append([1, shape, math.prod(shape)])
            layouts.append([tuple(run) for run in layout])
        self._graph_out_layouts = layouts

    def _unpack_graph_outputs(self):
        """Fresh output tensors: one clone per pack, then views (no further kernel launches)."""
        copies = [torch.empty(n, dtype=dtype, device=self.device) for n, dtype in self._graph_out_blocks]
        # one kernel for every output block (an SM copy: a cudaMemcpy D2D would queue on a copy engine
        # behind a concurrent download of the previous step's results); sources and sizes were marshalled
        # at capture time, only the fresh destinations are filled in
        backend = self.world._get_backend()
        bases = [c.data_ptr() for c in copies]
        for plan in self._graph_out_copy:
            backend.launches += plan.run(backend.lib, backend.device, bases)
        return self._views_of_output_blocks(copies)

    def _views_of_output_blocks(self, copies):
        """The step's output structure over freshly filled blocks (views only: no launches)."""
        fresh = [None] * len(self._graph_out_shapes)
        packs = self._graph_out_packs
        # leaves of equal shape that sit next to each other come out of ONE view + unbind
        for flat, (_, ids), layout in zip(copies, packs, self._graph_out_layouts):
            pieces = [flat] if len(layout) == 1 else flat.split_with_sizes([n * numel for n, _, numel in layout])
            k = 0
            for piece, (n, shape, _) in zip(pieces, layout):
                if n == 1:
                    fresh[ids[k]] = piece.view(shape)
                else:
                    for j, leaf in enumerate(piece.view((n,) + shape).unbind(0)):
                        fresh[ids[k + j]] = leaf
                k += n

        return _rebuild_outputs(self._graph_out_spec, fresh)

    def _capture(self, actions: List[Tensor]):
        if self.action_checks == "sync":
            raise RuntimeError("cuda_graph=True cannot be combined with action_checks='sync' (host sync per step)")
        if self.action_checks == "deferred" and self._bad_action_flag is None:
            self._bad_action_flag = torch.zeros(1, dtype=torch.bool, device=self.device)
        self._graph_action_layout = [(a.shape, a.dtype) for a in actions]
        dev_actions = [a.to(self.device) for a in actions]
        ingest_outside = self._fused_ingest_applies(
            [a.to(self._ingest_dtype()).contiguous() for a in dev_actions]
        )
        if ingest_outside:
            self._graph_inputs = None
        else:
            self._graph_inputs = [a.clone() for a in dev_actions]
        backend = self.world._get_backend()
        backend.refresh()
        backend.wait_for_jit()  # a run-time specialisation still compiling: capture the kernel that stays
        torch.cuda.synchronize(self.device)
        try:
            graph = torch.cuda.CUDAGraph(keep_graph=True)  # (the node count below needs the cudaGraph_t)
        except TypeError:  # pragma: no cover
            graph = torch.cuda.CUDAGraph()
        try:
            if ingest_outside:
                # (binds the action buffers; the replay that follows the capture ingests — and counts — again)
                self._apply_actions([a.to(self._ingest_dtype()).contiguous() for a in dev_actions], count_step=False)
            ingest_built_mask = bool(getattr(backend, "_mask_ready", False))
            before = backend.launches
            backend.trace = []
            with torch.cuda.graph(graph):
                # outputs stay un-cloned inside the graph; they are packed into flat buffers
                # there, and each replay hands out clones of those buffers
                if ingest_outside:
                    outputs = self._finish_step(True, clone_outputs=False)
                else:
                    outputs = self._step_device(self._graph_inputs, clone_outputs=False)
                self._pack_graph_outputs(outputs)
        except Exception as err:  # noqa: BLE001
            backend.trace = None
            raise RuntimeError(
                "cuda_graph=True: capturing Environment.step failed. The scenario (or a dynamics / "
                "action script) is not graph-safe: it must not synchronise with the host inside "
                f"process_action / pre_step / post_step / reward / observation / done / info. Cause: {err}"
            ) from err
        self._graph_launches = backend.launches - before
        backend.launches = before
        trace, backend.trace = backend.trace, None
        if hasattr(graph, "instantiate"):
            graph.instantiate()
        self._graph = graph
        self._graph_outputs = outputs
        self._graph_plan_version = self.world._plan_version
        self._one_call = None
        self._one_call_state = "off"
        if ingest_outside and _ONE_CALL_STEP:
            self._one_call = self._build_one_call_step(graph, ingest_built_mask, trace)
            # the first replay goes through torch and tells whether the graph draws device random numbers
            self._one_call_state = "probe" if self._one_call is not None else "off"

    def _library_only_step(self, graph, trace):
        """``(exact_broad_phase mode, program struct, StepProgram, plan, columns, obs block, limit)`` if the captured
        step consists of nothing but this library's ``World.step`` followed by one step program / observation
        launch — the graph then holds no torch kernel, and ``vmas_b200_env_step`` can issue those launches
        itself (direct mode), or one whole-step kernel.  ``limit``: ``(StepProgram, struct)`` of the environment's
        step limit if its launch follows (``_limit_program``), else None.  The observation launch may be followed by the
        plan's LIDAR launch (``backend.observe`` issues it from the same call, for exactly the plan's LIDAR terms).
        None otherwise."""
        kinds = None if trace is None else [t[0] for t in trace]
        if not _DIRECT_STEP or kinds not in (["step", "post"], ["step", "post", "post"]):
            return None
        (_, n_step, mode), (_, n_post, prog, plan, c, out) = trace[:2]
        limit, n_limit = None, 0
        if len(trace) == 3:
            _, n_limit, lprog, lplan, lc, _ = trace[2]
            own = getattr(self, "_limit_prog", None)
            if own is None or lprog is not own[1] or lplan is not None:
                return None  # (a second program of the scenario's)
            limit = (lprog, lc)
        values = plan is not None and bool(plan.buffer_sources)  # columns fed by the program: program, then gather
        lidars = plan is not None and bool(plan.compile(self.world)[1])
        n_want = (2 if values and prog is not None else 1) + (1 if lidars else 0)
        if n_post != n_want or n_step + n_post + n_limit != self._graph_launches:
            return None  # (anything else the backend launched)
        if values and any(not hasattr(src, "_slot") or src not in prog.outputs for src in plan.buffer_sources):
            return None  # (value columns that are not outputs of this program)
        backend = self.world._get_backend()
        try:
            nodes = backend.lib.vmas_b200_graph_num_nodes(graph.raw_cuda_graph())
        except Exception:  # noqa: BLE001  (no access to the cudaGraph_t: stay on the graph)
            return None
        if nodes != self._graph_launches:
            return None  # torch kernels / memsets in the graph: scenario code outside the program
        cols = None
        if plan is not None:
            dev = plan.device_cache.get(id(backend))
            # (a plan with LIDAR terms keeps its column table even without state columns: the whole-step kernel writes
            # the readings into its rows)
            cols = dev["cols"] if dev is not None and (dev["any_state"] or lidars) else None
        return mode, c, prog, plan, cols, out, limit

    def _splice_limit(self, c, prog, instrs, limit):
        """The scenario's program (struct ``c``, ``prog``, its resolved instructions ``instrs``) with the step limit
        ``limit = (StepProgram, struct)`` behind it as ONE program (``splice_program``): ``(struct, instructions,
        merged)``, ``merged.outputs`` the outputs of both with their slots in the merged program.  None if the result
        exceeds the program's registers, instructions or buffers, or ``terminated`` is not stored by ``prog``."""
        import types

        from ... import _native as N
        from .. import program as SP

        lprog, lc = limit
        feed_reg = None
        if lprog.feed_slot is not None:
            store_of = {b: a for op, _, a, b, _, _ in instrs if op in (SP.OP_STORE_F32, SP.OP_STORE_BOOL)}
            feed = lprog.resolve(lprog.buffers[lprog.feed_slot])
            o = next((o for o in prog.outputs if o.tensor is feed and o._slot in store_of), None)
            if o is None:
                return None
            feed_reg = store_of[o._slot]
        merged, n_regs, slots = splice_program(
            instrs, prog.n_regs, len(prog.buffers), lprog.instructions(None), lprog.feed_slot, feed_reg, lprog.count_slot
        )
        n_slots = len(prog.buffers) + len(slots)
        if n_regs > SP.MAX_REGS or len(merged) > N.PROG_MAX_INSTR or n_slots > N.PROG_MAX_BUFFERS:
            return None
        c2 = N.StepProgramC()
        ctypes.memmove(ctypes.addressof(c2), ctypes.addressof(c), ctypes.sizeof(c2))
        for k, (op, dst, a, b, arg, imm) in enumerate(merged):
            ins = c2.instr[k]
            ins.op, ins.dst, ins.a, ins.b, ins.arg, ins.imm = op, dst, a, b, arg, imm
        c2.n_instr = len(merged)
        outputs = list(prog.outputs)
        for old, new in slots.items():
            c2.buffers[new] = lc.buffers[old]
        for o in lprog.outputs:
            moved = SP.Output(o.dtype)
            moved.tensor, moved._slot = o.tensor, slots[o._slot]
            outputs.append(moved)
        return c2, merged, types.SimpleNamespace(outputs=outputs, buffers=[None] * n_slots)

    def _build_one_call_step(self, graph, ingest_built_mask: bool, trace=None):
        """Everything ``vmas_b200_env_step`` needs, marshalled once (None: this step does not fit the call)."""
        backend = self.world._get_backend()
        N = backend._native
        specs = self._fused_ingest_specs()
        live = [i for i, s in enumerate(specs) if s[0].action_size > 0]
        arr = getattr(backend, "_ingest_arr", None)
        if (
            arr is None or len(arr) != len(live) or not live or len(live) > N.MAX_INGEST_AGENTS
            or len(self._graph_out_copy) > 1 or len(self._graph_out_blocks) > N.MAX_OUT_BLOCKS
            or not hasattr(graph, "raw_cuda_graph_exec")
        ):
            return None
        counts = self.steps.dtype == torch.float32 and self.steps.is_contiguous()
        copy = self._graph_out_copy[0] if self._graph_out_copy else None
        items = [] if copy is None else [(src, block, offset) for src, (block, offset) in zip(copy.keep, copy.where)]
        direct = self._library_only_step(graph, trace)
        spliced = None
        if direct is not None and direct[6] is not None:
            # the step limit joins the scenario's program; the whole-step kernel takes its count from the prologue
            if counts:
                spliced = self._splice_limit(direct[1], direct[2], direct[2].instructions(backend.index_of), direct[6])
            if spliced is None:
                direct = None  # (too large a program, or no counter: the step stays on the graph)
        job, lidar_terms = None, []
        if direct is not None and direct[3] is not None:
            lidar_terms = direct[3].compile(self.world)[1]
        if direct is None:
            plan = N.EnvStepPlan(
                backend.lib, backend._dev_tables, self.world.slab, arr, len(live), self.clamp_action,
                self._bad_action_flag if self.action_checks == "deferred" else None, self.steps if counts else None,
                ingest_built_mask, graph.raw_cuda_graph_exec(), items, len(self._graph_out_blocks),
                block_kinds=self._graph_out_block_kinds,
            )
        else:
            mode, c, prog, oplan, cols, out, limit = direct
            instrs = prog.instructions(backend.index_of)
            merged = prog
            if spliced is not None:
                c, instrs, merged = spliced
            obs_to, mirrors = None, []
            if _WRITE_RESULTS_IN_PLACE:
                # results the post stage can write straight into the step's fresh blocks instead of into static
                # buffers that are then copied: the observation rows (if one leaf run covers the whole block),
                # and every leaf that is an output of the program (one more STORE per leaf)
                c, instrs, items, obs_to, mirrors = self._results_in_place(
                    c, merged, instrs, items, cols, out, self._graph_out_block_kinds
                )
            # the post stage rounds the observation rows itself where it writes them into the fresh block
            obs_dtype = N.DTYPE_F32 if obs_to is None else self._graph_out_block_kinds[obs_to[0]]
            plan = N.EnvStepPlan(
                backend.lib, backend._dev_tables, self.world.slab, arr, len(live), self.clamp_action,
                self._bad_action_flag if self.action_checks == "deferred" else None, self.steps if counts else None,
                ingest_built_mask, 0, items, len(self._graph_out_blocks), program=c, columns=cols,
                n_rows=0 if oplan is None else oplan.n_rows, width=0 if oplan is None else oplan.width, obs_out=out,
                exact_broad_phase=mode, obs_to=obs_to, mirrors=mirrors, block_kinds=self._graph_out_block_kinds,
                obs_dtype=obs_dtype,
            )
            plan.keep += (prog, oplan, limit)
            if _WHOLE_STEP_KERNEL and backend._dev_tables.tb.specialization >= 0:
                # the whole-step kernel of this (world, program, observation plan): compiled once (seconds),
                # cached on disk; until it is there the step runs as two launches — same bits
                from ... import codegen, jit

                cols_np = None if cols is None else oplan.compile(self.world)[0]
                if cols_np is not None:
                    cols_np = codegen.fuse_value_columns(cols_np, oplan.buffer_sources, instrs)
                # ... with the action ingest (and the broad phase) as its prologue where the agents allow it
                # (codegen.prologue_acts: their action models; static agents have nothing to ingest): the whole
                # step is then ONE launch.  Continuous, discrete and multi-discrete spaces alike.
                acts = ()
                if (
                    _INGEST_IN_KERNEL
                    and type(self.scenario).pre_step is BaseScenario.pre_step and not self.world.scripted_agents
                    and (ingest_built_mask or backend.tables.n_masked == 0 or not self.world.exact_broad_phase)
                ):
                    acts = codegen.prologue_acts(arr, N.ACT_CONTINUOUS if self.continuous_actions else int(arr[0].action_kind))
                    if acts:
                        plan.c.ingest_in_kernel = 1
                # the plan's LIDARs are cast in the kernel's epilogue (None: a sensor sees more targets than it takes)
                lidar = codegen.lidar_sensors(lidar_terms, backend.index_of, backend.ray_targets) if lidar_terms else None
                if lidar is not None or not lidar_terms:
                    job = jit.request_step_kernel(backend.tables.desc, cols_np, instrs, acts, obs_dtype=obs_dtype,
                                                  lidar=lidar)
                if job is not None:
                    job.done.wait(timeout=_WHOLE_STEP_KERNEL_WAIT_S)
            plan.measurements = self._lidar_measurements(lidar_terms, obs_to, oplan)
        if direct is not None and direct[3] is not None and (direct[3].buffer_sources or lidar_terms) and not (
            job is not None and job.done.is_set() and job.index > 0
        ):
            # value columns need the program and the gather in ONE thread, and the direct launches have no LIDAR
            # launch: without the whole-step kernel the step stays a captured graph (program launch, then gather
            # launch, then the LIDAR launch)
            return self._build_one_call_step(graph, ingest_built_mask, None)
        plan.direct = direct is not None
        plan.job = job
        plan.live = live
        plan.bind = [(agent.action, u) for agent, _, u in specs]
        plan.counts = counts
        plan.drones = list(getattr(backend, "_ingest_drones", []))
        self._adopt_whole_step_kernel(plan)
        return plan

    def _results_in_place(self, c, prog, instrs, items, cols, out, block_kinds=None):
        """Splits the hand-out copies ``items`` = [(source, block, byte offset)] into what the post stage can
        write in place.  ``block_kinds[b]``: ``DTYPE_F16`` / ``DTYPE_BF16`` if block ``b`` receives its fp32
        sources rounded to 16 bits (the observation rows are then written in place as such; no program store is
        mirrored into it).  Returns ``(program struct with the extra stores, its instructions, the copies that
        remain, (block, offset) of the observation rows or None, [(buffer slot, block, offset)])``."""
        from ... import _native as N
        from .. import program as SP

        B = self.num_envs
        by_ptr = {}
        for o in prog.outputs:
            by_ptr.setdefault((o.tensor.data_ptr(), o.tensor.dtype), o)
        store_of = {}  # output slot -> register it stores
        for op, dst, a, b, arg, imm in instrs:
            if op in (SP.OP_STORE_F32, SP.OP_STORE_BOOL):
                store_of[b] = (op, a)
        rest, obs_to, mirrors, extra = [], None, [], []
        n_slots = len(prog.buffers)
        obs_pieces = set()
        if cols is not None and out is not None:
            # the copies that together move the observation block, piece after piece, to one place
            lo, size = out.data_ptr(), out.numel() * out.element_size()
            inside = [k for k, (src, _, _) in enumerate(items) if lo <= src.data_ptr() < lo + size]
            if inside:
                _, block0, offset0 = items[inside[0]]
                shrink = 2 if block_kinds and block_kinds[block0] else 1  # (fp32 rows land as 16-bit values)
                at = 0
                for k in inside:
                    src, block, offset = items[k]
                    if src.data_ptr() != lo + at or block != block0 or offset != offset0 + at // shrink:
                        break
                    at += src.numel() * src.element_size()
                else:
                    if at == size and offset0 % 16 == 0:
                        obs_to, obs_pieces = (block0, offset0), set(inside)
        for k, (src, block, offset) in enumerate(items):
            if k in obs_pieces:
                continue
            o = by_ptr.get((src.data_ptr(), src.dtype))
            if (
                o is not None and src.numel() == B and o._slot in store_of and not (block_kinds and block_kinds[block])
                and n_slots + len(extra) < N.PROG_MAX_BUFFERS and len(instrs) + len(extra) < N.PROG_MAX_INSTR
            ):
                op, reg = store_of[o._slot]
                slot = n_slots + len(extra)
                extra.append((op, 0, reg, slot, 0, 0.0))
                mirrors.append((slot, block, offset))
                continue
            rest.append((src, block, offset))
        if not extra:
            return c, instrs, rest, obs_to, mirrors
        c2 = N.StepProgramC()
        ctypes.memmove(ctypes.addressof(c2), ctypes.addressof(c), ctypes.sizeof(c2))
        for k, (op, dst, a, b, arg, imm) in enumerate(extra):
            ins = c2.instr[len(instrs) + k]
            ins.op, ins.dst, ins.a, ins.b, ins.arg, ins.imm = op, dst, a, b, arg, imm
        c2.n_instr = len(instrs) + len(extra)
        return c2, instrs + extra, rest, obs_to, mirrors

    def _lidar_measurements(self, lidar_terms, obs_to, oplan):
        """What a one-call step makes of ``Lidar._last_measurement``: None when the readings land where the graph
        path put them (the static observation block), else ``(block, first element, shape, [(sensor, row, column,
        rays)])`` of the readings in the step's fresh result block.  In an fp32 block an unflipped sensor's entry is
        a view of its readings, as ``backend.observe`` leaves it; a flipped sensor gets None, as there.  A 16-bit
        block holds no fp32 readings: every sensor gets None."""
        if not lidar_terms or obs_to is None:
            return None
        block, offset = obs_to
        fp32 = not self._graph_out_block_kinds[block]
        sensors = [(s, r, c, int(s._angles.shape[1]) if fp32 and not flipped else 0) for r, c, s, flipped in lidar_terms]
        return block, offset // 4 if fp32 else None, (oplan.n_rows, self.num_envs, oplan.width), sensors

    def _adopt_whole_step_kernel(self, plan):
        job = plan.job
        if job is None or not job.done.is_set():
            return
        plan.job = None
        if job.index > 0:
            plan.c.fused_kernel = job.index
        elif job.error:
            import warnings

            warnings.warn(f"vmas_b200: no whole-step kernel, staying on two launches per step ({job.error})")

    def _step_one_call(self, actions: List[Tensor]):
        """A captured step through ``vmas_b200_env_step``: action ingest, graph launch and the hand-out copy
        in one crossing of the FFI."""
        plan = self._one_call
        if plan.job is not None:
            self._adopt_whole_step_kernel(plan)
        agents = plan.agents
        for k, i in enumerate(plan.live):
            agents[k].actions = actions[i].data_ptr()
        for c, model in plan.drones:  # a reset re-binds the drone's 12-state tensor
            c.dyn_state = model.drone_state.data_ptr()
        device = self.device
        copies = [torch.empty(n, dtype=dtype, device=device) for n, dtype in self._graph_out_blocks]
        blocks = plan.out_blocks
        for j, c in enumerate(copies):
            blocks[j] = c.data_ptr()
        launched = plan.run()  # (the kernels the call issued itself; a graph's nodes come on top)
        measured = getattr(plan, "measurements", None)
        if measured is not None:
            block, first, shape, sensors = measured
            rows = None if first is None else copies[block][first : first + math.prod(shape)].view(shape)
            for sensor, r, c, n in sensors:
                sensor._last_measurement = rows[r, :, c : c + n] if n else None
        for action, u in plan.bind:  # (a reset replaces agent.action.u; the call writes the static buffers)
            if action._u is not u:
                action.u = u
        self.graph_replays += 1
        backend = self.world._get_backend()
        backend.launches += launched + (0 if plan.direct else self._graph_launches)
        backend._mask_ready = False
        backend.after_step()
        return self._views_of_output_blocks(copies)

    def _done(self, clone=True):
        terminated = self.scenario.done()
        limit = self._limit_applies(terminated)
        if limit is not None:
            # the step limit as a step program: one library launch (and, captured, part of the whole-step kernel)
            self._limit_input = terminated
            limit.run()
            out = limit.out.tensor
            if clone:
                terminated, out = terminated.clone(), out.clone()
            return (terminated, out) if self.terminated_truncated else out
        if clone:
            terminated = terminated.clone()
        truncated = self.steps >= self.max_steps if self.max_steps is not None else None
        if self.terminated_truncated:
            if truncated is None:
                truncated = torch.zeros_like(terminated)
            return terminated, truncated
        if truncated is None:
            return terminated
        return terminated + truncated

    def _limit_program(self):
        """``max_steps`` and the terminated / truncated split as a step program of the environment's own: the same
        statements as ``_done``'s torch ops, bit for bit (``steps >= max_steps`` compares in fp32, as torch does with
        an fp32 counter).  ``.out`` is ``dones`` (``terminated_truncated=False``) or ``truncated``.  Built again when
        the limit changes; a captured step keeps the one it was captured with."""
        from .. import program as SP

        key = (self.max_steps, self.terminated_truncated)
        cached = getattr(self, "_limit_prog", None)
        if cached is not None and cached[0] == key and cached[1].world is self.world:
            return cached[1]
        p = SP.StepProgram(self.world)
        p.count_slot = p.feed_slot = None  # buffer slots of the counter and of terminated (_splice_limit)
        if self.max_steps is None:
            p.out = p.store(p.const(0.0), torch.bool)
        else:
            count = p.load(lambda: self.steps)
            p.count_slot = len(p.buffers) - 1
            truncated = p.le(p.const(float(self.max_steps)), count)
            if not self.terminated_truncated:
                terminated = p.load(lambda: self._limit_input, is_bool=True)
                p.feed_slot = len(p.buffers) - 1
                truncated = p.logical_or(terminated, truncated)
            p.out = p.store(truncated, torch.bool)
        p.finalize()
        self._limit_prog = (key, p)
        return p

    def _limit_applies(self, terminated):
        """The limit program if ``_done`` runs it in place of its torch ops: on CUDA, inside a step (no auto-reset),
        for a limit or a split, when ``terminated`` is an output of a step program of this step.  None otherwise."""
        if self.max_steps is None and not self.terminated_truncated:
            return None
        programs = getattr(self.world._get_backend(), "step_programs", None)
        if not programs or self.steps.dtype != torch.float32 or not self.steps.is_contiguous():
            return None
        if not any(o.tensor is terminated and o.dtype == torch.bool for prog in programs for o in prog.outputs):
            return None
        return self._limit_program()

    # ------------------------------------------------------------------------------------
    # spaces
    # ------------------------------------------------------------------------------------
    def get_action_space(self):
        if self.dict_spaces:
            return spaces.Dict({a.name: self.get_agent_action_space(a) for a in self.agents})
        return spaces.Tuple([self.get_agent_action_space(a) for a in self.agents])

    def get_observation_space(self, observations: Union[List, Dict]):
        if self.dict_spaces:
            return spaces.Dict(
                {
                    a.name: self.get_agent_observation_space(a, observations[a.name])
                    for a in self.agents
                }
            )
        return spaces.Tuple(
            [self.get_agent_observation_space(a, observations[i]) for i, a in enumerate(self.agents)]
        )

    def _comm_dims(self, agent: Agent) -> int:
        return self.world.dim_c if not agent.silent else 0

    def get_agent_action_size(self, agent: Agent):
        if self.continuous_actions:
            return agent.action.action_size + self._comm_dims(agent)
        if self.multidiscrete_actions:
            return agent.action_size + (1 if self._comm_dims(agent) != 0 else 0)
        return 1

    def get_agent_action_space(self, agent: Agent):
        comm = self._comm_dims(agent)
        if self.continuous_actions:
            u_range = agent.action.u_range_tensor.tolist()
            return spaces.Box(
                low=np.array([-r for r in u_range] + [0] * comm, dtype=np.float32),
                high=np.array(u_range + [1] * comm, dtype=np.float32),
                shape=(self.get_agent_action_size(agent),),
                dtype=np.float32,
            )
        if self.multidiscrete_actions:
            return spaces.MultiDiscrete(list(agent.discrete_action_nvec) + ([comm] if comm != 0 else []))
        return spaces.Discrete(math.prod(agent.discrete_action_nvec) * (comm if comm != 0 else 1))

    def get_agent_observation_space(self, agent: Agent, obs: AGENT_OBS_TYPE):
        if isinstance(obs, Tensor):
            # obs_dtype=torch.bfloat16: numpy has no bfloat16, the space stays fp32
            dtype = np.float16 if self.obs_dtype == torch.float16 else np.float32
            return spaces.Box(low=-dtype("inf"), high=dtype("inf"), shape=obs.shape[1:], dtype=dtype)
        if isinstance(obs, Dict):
            return spaces.Dict(
                {k: self.get_agent_observation_space(agent, v) for k, v in obs.items()}
            )
        raise NotImplementedError(f"Invalid type of observation {obs} for agent {agent.name}")

    # ------------------------------------------------------------------------------------
    # random actions (ref environment.py:525-607)
    # ------------------------------------------------------------------------------------
    @_seeded
    def get_random_action(self, agent: Agent) -> Tensor:
        """A uniformly random valid action ``[batch_dim, action_size]`` for ``agent``."""
        kw = dict(device=agent.device, dtype=torch.float32)
        if self.continuous_actions:
            cols = []
            for k in range(agent.action_size):
                r = agent.action.u_range_tensor[k]
                cols.append(torch.zeros(agent.batch_dim, **kw).uniform_(-r, r))
            for _ in range(self._comm_dims(agent)):
                cols.append(torch.zeros(agent.batch_dim, **kw).uniform_(0, 1))
            return torch.stack(cols, dim=-1)
        space = self.get_agent_action_space(agent)
        if self.multidiscrete_actions:
            cols = [
                torch.randint(low=0, high=int(n), size=(agent.batch_dim,), device=agent.device)
                for n in space.nvec
            ]
            return torch.stack(cols, dim=-1)
        return torch.randint(low=0, high=int(space.n), size=(agent.batch_dim,), device=agent.device)

    def get_random_actions(self) -> Sequence[Tensor]:
        """Random actions for all policy agents, ready for :meth:`step`."""
        return [self.get_random_action(agent) for agent in self.agents]

    # ------------------------------------------------------------------------------------
    # action decoding (ref environment.py:609-749)
    # ------------------------------------------------------------------------------------
    def _flag_if(self, condition: Tensor, message: str):
        """``assert not condition.any()`` — immediately, deferred to the next call, or never."""
        if self.action_checks == "off":
            return
        if self.action_checks == "sync":
            assert not bool(condition.any()), message
            return
        if self._bad_action_flag is None:
            self._bad_action_flag = torch.zeros(1, dtype=torch.bool, device=self.device)
        self._bad_action_flag |= condition.any()
        if message not in self._bad_action_messages:
            self._bad_action_messages.append(message)

    #: deferred action checks copy their (sticky) device flag to the host every this many steps
    ACTION_READBACK_EVERY = 8

    def _launch_deferred_action_readback(self, force: bool = False):
        if self.action_checks != "deferred" or self._bad_action_flag is None:
            return
        # the device flag is sticky: looking at it every few steps loses nothing
        self._readback_tick = getattr(self, "_readback_tick", 0) + 1
        if self._bad_action_host is not None and self._readback_tick % self.ACTION_READBACK_EVERY and not force:
            return
        if self._bad_action_host is None:
            pin = self.device.type == "cuda"
            self._bad_action_host = torch.zeros(1, dtype=torch.bool, pin_memory=pin)
            self._bad_action_event = torch.cuda.Event() if pin else None
        elif self._bad_action_event is not None and not self._bad_action_event.query():
            return  # the previous read-back is still in flight; the flag is sticky, nothing is lost
        self._bad_action_host.copy_(self._bad_action_flag, non_blocking=True)
        self._readback_pending = True
        if self._bad_action_event is not None:
            self._bad_action_event.record()

    def _raise_deferred_action_errors(self, wait: bool = False):
        """Raises if a previous step flagged an invalid action.  Never stalls the pipeline: the
        flag is looked at only once its asynchronous read-back has landed (``wait=True`` forces it)."""
        if self._bad_action_host is None or not getattr(self, "_readback_pending", False):
            return
        if self._bad_action_event is not None:
            if wait:
                self._bad_action_event.synchronize()
            elif not self._bad_action_event.query():
                return
        self._readback_pending = False  # the copy has landed: look at it once
        if bool(self._bad_action_host.item()):
            self._bad_action_flag.zero_()
            self._bad_action_host.zero_()
            raise AssertionError(
                "Invalid action in the previous step: " + "; ".join(self._bad_action_messages)
            )

    def check_actions_now(self):
        """Force the deferred action checks to be read back and raised (one host sync)."""
        self._launch_deferred_action_readback(force=True)
        self._raise_deferred_action_errors(wait=True)

    def _check_discrete_action(self, action: Tensor, low: int, high: int, type: str):
        self._flag_if(
            (action < low) | (action >= high),
            f"Discrete {type} actions are out of bounds, allowed int range [{low},{high})",
        )

    def _set_action(self, action: Tensor, agent: Agent):
        action = action.detach().to(self.device)
        self._flag_if(action.isnan(), f"Action of agent {agent.name} contains NaN")
        assert action.shape[1] == self.get_agent_action_size(agent), (
            f"Agent {agent.name} has wrong action size, got {action.shape[1]}, "
            f"expected {self.get_agent_action_size(agent)}"
        )
        n_phys = agent.action_size
        comm = self._comm_dims(agent)
        u_range = agent.action.u_range_tensor

        if self.clamp_action and self.continuous_actions:
            physical = action[..., :n_phys].clamp(-u_range, u_range)
            if comm > 0:
                action = torch.cat([physical, action[..., n_phys:].clamp(0, 1)], dim=-1)
            else:
                action = physical

        column = 0
        if self.continuous_actions:
            physical = action[:, :n_phys]
            column += self.world.dim_p
            self._flag_if(
                torch.abs(physical) > u_range,
                f"Physical actions of agent {agent.name} are out of its range {agent.u_range}",
            )
            u = physical.to(torch.float32).clone()
        else:
            action = action.clone()
            if not self.multidiscrete_actions:
                # unravel the flat index of the cartesian product into one index per component
                flat = action.squeeze(-1)
                nvec = list(agent.discrete_action_nvec) + ([self.world.dim_c] if comm != 0 else [])
                parts = []
                for i in range(len(nvec)):
                    stride = math.prod(nvec[i + 1 :])
                    parts.append(flat // stride)
                    flat = flat % stride
                action = torch.stack(parts, dim=-1)
            u = torch.zeros(self.batch_dim, n_phys, device=self.device, dtype=torch.float32)
            for n in agent.discrete_action_nvec:
                idx = action[:, column]
                self._check_discrete_action(idx.unsqueeze(-1), low=0, high=n, type="physical")
                u_max = u_range[column]
                if n % 2 != 0:
                    # odd n: index 0 means "no force"; indices 1..n//2 shift down by one
                    stay = idx == 0
                    lower_half = (idx > 0) & (idx <= n // 2)
                    idx = torch.where(stay, torch.full_like(idx, n // 2), idx)
                    idx = torch.where(lower_half, idx - 1, idx)
                u[:, column] = (idx / (n - 1)) * (2 * u_max) - u_max
                column += 1

        u = u * agent.action.u_multiplier_tensor
        noise_level = agent.action.u_noise
        if (max(noise_level) if isinstance(noise_level, Sequence) else noise_level) > 0:
            u = u + torch.randn(*u.shape, device=self.device, dtype=torch.float32) * agent.action.u_noise_tensor
        agent.action.u = u

        if comm > 0:
            comm_action = action[:, column:]
            if not self.continuous_actions:
                self._check_discrete_action(comm_action, 0, self.world.dim_c, "communication")
                one_hot = torch.zeros(
                    self.num_envs, self.world.dim_c, device=self.device, dtype=torch.float32
                )
                one_hot.scatter_(1, comm_action.long(), 1)
                c = one_hot
            else:
                self._flag_if(
                    (comm_action > 1) | (comm_action < 0), "Comm actions are out of range [0,1]"
                )
                c = comm_action.clone()
            if agent.c_noise > 0:
                c = c + torch.randn(*c.shape, device=self.device, dtype=torch.float32) * agent.c_noise
            agent.action.c = c

    # ------------------------------------------------------------------------------------
    def render(self, *args, **kwargs):
        raise NotImplementedError(
            "Rendering (pyglet viewer) is outside the scope of the CUDA hot-path build"
        )

    def to(self, device: DEVICE_TYPING):
        device = torch.device(device)
        self.scenario.to(device)
        super().to(device)
