"""Test-only stand-in for ``gym`` so the UNMODIFIED reference imports without
gym installed (it needs ``gym.Env`` and ``gym.spaces``).  Never imported by the product package."""
from . import spaces  # noqa: F401


class Env:
    metadata = {}


class Wrapper(Env):
    def __init__(self, env=None):
        self.env = env
