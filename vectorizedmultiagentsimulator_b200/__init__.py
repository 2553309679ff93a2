"""vectorizedmultiagentsimulator_b200 — an H100-native drop-in for VMAS's physics hot path.

``World.step`` (batched 2-D rigid-body substep: forces, Sphere/Box/Line contacts, joints,
semi-implicit Euler) and the LIDAR ray cast are hand-written sm_90a CUDA kernels behind the
reference's own Python API (``make_env`` / ``Environment.step`` / ``BaseScenario``).
"""
from .make_env import make_env
from .simulator.environment import Environment, Wrapper

__version__ = "0.1.0"

__all__ = ["make_env", "Environment", "Wrapper", "scenarios", "stack_views"]


def stack_views(tensors):
    """``torch.stack(tensors)`` without the copy where none is needed.

    ``Environment.step`` hands out the per-agent results of a step (observations, rewards) as slices that sit
    back to back in one freshly filled block; code that wants them as ONE tensor — to send them to the host in
    a single transfer, say — gets a ``[n, ...]`` view of that block here, and a plain ``torch.stack`` copy for
    any other list of tensors."""
    import torch

    first = tensors[0]
    nbytes = first.numel() * first.element_size()
    base = first.untyped_storage().data_ptr() if first.numel() else 0
    if nbytes and all(
        t.shape == first.shape and t.dtype == first.dtype and t.device == first.device and t.is_contiguous()
        and t.untyped_storage().data_ptr() == base and t.data_ptr() == first.data_ptr() + i * nbytes
        for i, t in enumerate(tensors)
    ):
        return first.as_strided((len(tensors),) + tuple(first.shape), (first.numel(),) + tuple(first.stride()))
    return torch.stack(list(tensors))

#: scenarios shipped with this build (re-written on the public API; same names as the reference)
scenarios_list = ["balance", "flocking", "navigation", "transport"]
