"""PID velocity controller: turns a velocity target in ``agent.action.u`` into a force
(API and arithmetic of ref vmas/simulator/controllers/velocity_controller.py:16-125).

``ctrl_params`` is ``[gain, integral time, derivative time]`` in ``"standard"`` form or
``[kP, kI, kD]`` in ``"parallel"`` form (``Ti = kP / kI``, ``Td = kD / kP``).  On a CUDA world
``process_force`` is one kernel launch (``vmas_b200_velocity_controller``: the same fp32 statements in
the same order); elsewhere (the CPU oracle backend of the tests) the torch ops below.
"""
from __future__ import annotations

import warnings
from typing import Optional

import torch


class VelocityController:
    def __init__(self, agent, world, ctrl_params=(1, 0, 0), pid_form: str = "standard"):
        self.agent = agent
        self.world = world
        self.dt = world.dt
        self.ctrl_gain = ctrl_params[0]
        if pid_form == "standard":
            self.integralTs, self.derivativeTs = ctrl_params[1], ctrl_params[2]
        elif pid_form == "parallel":
            self.integralTs = 0.0 if ctrl_params[1] == 0 else self.ctrl_gain / ctrl_params[1]
            self.derivativeTs = ctrl_params[2] / self.ctrl_gain
        else:
            raise Exception("PID form is either standard or parallel.")

        self.use_integrator = self.integralTs != 0
        if self.use_integrator:
            # anti-windup at half of the tighter force limit
            limits = [x for x in (agent.max_f, agent.f_range) if x is not None]
            if limits:
                fmax = min(limits)
                self.integrator_windup_cutoff = 0.5 * fmax * self.integralTs / (self.dt * self.ctrl_gain)
            else:
                self.integrator_windup_cutoff = None
                warnings.warn("Force limits not specified. Integrator can wind up!")
        self.reset()

    def reset(self, index: Optional[int] = None):
        if index is None:
            shape = (self.world.batch_dim, self.world.dim_p)
            self.accum_errs = torch.zeros(shape, device=self.world.device)
            self.prev_err = torch.zeros(shape, device=self.world.device)
        else:
            self.accum_errs = self.accum_errs.clone()
            self.prev_err = self.prev_err.clone()
            self.accum_errs[index] = 0.0
            self.prev_err[index] = 0.0

    def integralError(self, err):
        if not self.use_integrator:
            return 0
        self.accum_errs += self.dt * err
        if self.integrator_windup_cutoff is not None:
            self.accum_errs = self.accum_errs.clamp(
                -self.integrator_windup_cutoff, self.integrator_windup_cutoff
            )
        return (1.0 / self.integralTs) * self.accum_errs

    def rateError(self, err):
        rate = self.derivativeTs * (err - self.prev_err) / self.dt
        self.prev_err = err
        return rate

    #: tests set this to False to run the torch statements on CUDA too (the kernel is compared with them)
    use_kernel = True

    def _process_force_cuda(self) -> bool:
        """The fused path: needs a CUDA world on this package's backend and a contiguous [B, 2] action."""
        world, agent = self.world, self.agent
        backend = world._get_backend() if hasattr(world, "_get_backend") else None
        u = agent.action.u
        if (
            not self.use_kernel or backend is None or not hasattr(backend, "lib") or u is None or u.device.type != "cuda"
            or u.dim() != 2 or u.shape[1] != 2 or not u.is_contiguous() or u.dtype != torch.float32
        ):
            return False
        self.accum_errs = self.accum_errs.to(world.device).contiguous()
        self.prev_err = self.prev_err.to(world.device).contiguous()
        backend.refresh()
        cutoff = getattr(self, "integrator_windup_cutoff", None)
        backend.launches += backend._native.velocity_controller(
            backend.lib, backend._dev_tables, world.slab, backend.index_of(agent), u, self.accum_errs, self.prev_err,
            self.ctrl_gain, (1.0 / self.integralTs) if self.use_integrator else 0.0, self.derivativeTs, self.dt,
            -1.0 if cutoff is None else cutoff, agent.mass,
        )
        return True

    def process_force(self):
        if isinstance(self.agent.mass, torch.Tensor) and self.agent.mass.dim() > 0:
            raise NotImplementedError(
                f"Entity '{self.agent.name}': a per-env mass on an agent driven by the velocity controller is out of scope"
            )
        if self._process_force_cuda():
            return
        self.accum_errs = self.accum_errs.to(self.world.device)
        self.prev_err = self.prev_err.to(self.world.device)
        err = self.agent.action.u - self.agent.state.vel
        u = self.ctrl_gain * (err + self.integralError(err) + self.rateError(err))
        u *= self.agent.mass
        self.agent.action.u = u
