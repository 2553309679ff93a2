"""CPU ORACLE for the CUDA physics hot path — TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A torch-fp32, CPU-only restatement of the reference's ``World.step``, LIDAR ray cast and
distance queries (``vmas/simulator/{core,physics,joints}.py``), used as the
checker the CUDA kernels are compared against.

Parity status: PINNED — validated against the unmodified reference's recorded roll-outs
(``tests/test_oracle_vs_reference.py``) and against committed golden roll-outs generated from
the reference (``tests/golden/``, made by ``tests/make_golden.py``).

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline legs may import
this package.  Nothing under ``vectorizedmultiagentsimulator_b200/`` imports it.
"""
