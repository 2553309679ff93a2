"""How much can sorting envs by contact signature reduce a warp's divergent work?  (CPU study: real roll-out
states from the oracle env, signatures from the specialised kernel's device code run on the host, tests/hostsim.)

    python tools/grouping_study.py
"""
import os, sys, ctypes as C, numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))
import vectorizedmultiagentsimulator_b200 as b200
from oracle.backend import use_oracle
from vectorizedmultiagentsimulator_b200 import codegen
from vectorizedmultiagentsimulator_b200.simulator import plan as P
import test_hostsim as TH
TH._build()
lib = C.CDLL(TH.SIM_LIB)
lib.hostsim_step.argtypes = [C.c_uint64, C.c_int, C.c_int] + [C.c_void_p] * 7 + [C.c_int] * 3
lib.hostsim_record_signatures.argtypes=[C.c_void_p]
def study(name, kwargs, B=4096, steps=60):
    torch.manual_seed(0)
    with use_oracle():
        env = b200.make_env(name, num_envs=B, device="cpu", seed=0, **kwargs)
        for t in range(steps):
            env.step(env.get_random_actions())
        # state right before the next world.step: apply actions
        acts = env.get_random_actions()
        env._apply_actions(acts) if hasattr(env,'_apply_actions') else None
    w = env.world
    desc = P.describe_world(w); h = codegen.world_hash(desc)
    slab = w.slab
    arr = {k: np.ascontiguousarray(getattr(slab,k).numpy().astype(np.float32)).copy() for k in ("pos","vel","rot","ang_vel","force","torque")}
    sig = np.zeros(B, np.uint32)
    lib.hostsim_record_signatures(sig.ctypes.data)
    rc = lib.hostsim_step(h, 0, B, *(arr[k].ctypes.data for k in ("pos","vel","rot","ang_vel","force","torque")), None, 0, 0, desc.substeps)
    assert rc == 0
    pc = np.array([bin(x).count("1") for x in sig])
    print(f"{name}: live items per env {pc.mean():.2f}, distinct signatures {len(set(sig.tolist()))}")
    for win in (32, 256, 512, 2048, B):
        order = np.arange(B)
        if win > 32:
            for lo in range(0, B, win):
                idx = np.arange(lo, min(B, lo+win))
                order[lo:lo+len(idx)] = idx[np.argsort(sig[idx], kind="stable")]
        s = sig[order].reshape(-1, 32)
        union = np.array([bin(int(np.bitwise_or.reduce(r))).count("1") for r in s])
        lanes = np.array([sum(bin(int(x)).count("1") for x in r) for r in s]) / np.maximum(union,1)
        print(f"   sort window {win:5d}: items live in any lane of a warp {union.mean():5.2f}  (avg lanes active in those {lanes.mean():5.1f})")
study("balance", dict(n_agents=4))
study("flocking", dict(n_agents=5))
