"""oracle/ -- TEST INFRASTRUCTURE ONLY.

CPU restatement (numpy / torch-fp32 / plain C) of DF-VO's per-frame tracking hot path,
used exclusively as the *checker* for the CUDA path:

  * only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` /
    ``--impl reference`` legs may import anything from this package;
  * nothing under ``df-vo_b200/`` (the product) imports it, and the product raises if the
    CUDA library is missing instead of falling back to this code.

Pinning status: the reference repository ships no tests, golden vectors or weights
(SURVEY.md section 4), so the oracle is pinned against *outputs of the reference itself*
(``oracle/gen_golden.py`` imports a DF-VO checkout named by ``DFVO_REFERENCE_ROOT`` under
``oracle/shims.py`` and writes ``tests/golden/*.npz``), and against the third-party
solvers the reference calls (``cv2`` 4.13.0, ``sklearn`` 1.9.0), which the tests import too.  See DESIGN.md "Oracle" for the per-function table.
"""
