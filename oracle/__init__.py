"""CPU oracle for the torchcde hot path.  TEST INFRASTRUCTURE ONLY.

Nothing under ``oracle/`` is part of the product.  Only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline / ``--impl reference``
legs may import it, and there only as the checker or the timed CPU arm -- never as
a fallback for the CUDA path (``torchcde_b200`` raises when its CUDA library is
missing; it never routes here).

Pinning status (see DESIGN.md "Oracle"):
  * path (i)  coefficient construction + spline evaluation: PINNED.  Every function is
    checked bit-for-bit against the live reference (imported from its checkout with
    the two absent solver packages stubbed, ``oracle/reference_loader.py``) and against
    the reference tests' own known-answer vectors; the generated vectors are committed
    under ``tests/golden/`` by ``oracle/make_golden.py``.
  * path (ii) fixed-step solve: the vector field is PINNED against the reference's own
    ``_VectorField.forward`` (solver.py:117-135); the time stepping is a restatement of
    torchdiffeq's published fixed-grid algorithm (third-party, constraint
    ``torchdiffeq>=0.2.0`` at setup.py:51, absent from this machine).  For the stepping
    arithmetic itself: PARITY UNPINNED against a torchdiffeq binary; it is anchored
    on analytic solutions derived from the reference's own test fixtures
    (test_cdeint.py:54-55, :90-95), on convergence order, and on the reference
    ``cdeint`` call site being executed end-to-end with the port plugged in where
    torchdiffeq would be.
"""
