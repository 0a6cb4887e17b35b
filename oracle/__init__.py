"""CPU oracle for the vMAP vectorised per-object training step.

TEST INFRASTRUCTURE ONLY.  Nothing under ``oracle/`` is part of the product:
only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s
``cpu_baseline`` / ``--impl reference`` legs may import it, and only as the
checker / the timed CPU baseline -- never as a fallback for the CUDA path.

Parity pinning: the reference (kxhit/vMAP) ships no tests, golden vectors or
seeds (SURVEY.md section 4), so the restatement here is pinned against outputs
of the reference's *own modules* imported from a reference checkout
(``oracle/_refload.py``): ``oracle/make_golden.py`` and
``oracle/make_reference_golden.py`` generate ``tests/golden/*.npz``, and
``tests/test_oracle_golden.py`` / ``tests/test_oracle_live_reference.py``
replay them on any machine.
"""
