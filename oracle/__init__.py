"""TEST INFRASTRUCTURE — CPU restatements of the reference's algorithms for the hot path.

Nothing in the shipped package (``abr_control_b200``) imports this package; only ``tests/``,
``__graft_entry__.smoke()`` and the CPU-baseline / ``--impl reference`` legs of ``bench.py`` may import, link or execute
anything below ``oracle/`` (tests/test_abi.py::test_package_does_not_import_the_oracle enforces the first part).

* ``rbd_oracle.py``  rigid-body quantities by the literal product rule over the chain factors
* ``osc_oracle.py``  ``OSC.generate`` and the other controllers with the reference's own NumPy calls
* ``ik_oracle.py``   the inverse-kinematics planner's iteration
* ``ctrl_batch.py``  batched restatements of ``Joint``, ``Floating``, ``Sliding`` and the IK iteration, with per-state
                     conditioning flags
* ``c/``             C restatement of the NumPy half of ``OSC.generate`` (for the multi-threaded CPU baseline)
* ``ref_harness/``   runs the REFERENCE in the development container and writes ``tests/golden/*.npz``
* ``_ref/``          (git-ignored) the reference's own generated C for UR5, compiled where the reference wrote it

Every restatement is pinned against those goldens (tests/test_oracle_golden.py).
"""
