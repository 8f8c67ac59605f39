"""TEST INFRASTRUCTURE ONLY — CPU restatement ("oracle") of the ControlAR conditional-decoding hot path.

Nothing under ``oracle/`` is part of the product.  Only ``tests/``, ``__graft_entry__.smoke()`` and the
``cpu_baseline`` / ``--impl reference`` legs of ``bench.py`` may import it, and there only as the checker
(or as the timed CPU baseline), never as the thing shipped.  The product path (``controlar_b200``) never
imports this package and fails loudly when its CUDA library is missing.

Parity pinning: the restatement is checked against outputs of the *reference itself* (the Python modules of a
reference checkout, imported read-only) by ``tests/golden/make_golden.py``; the resulting
vectors are committed under ``tests/golden/*.pt`` and ``tests/test_oracle_golden.py`` replays them.  The
reference ships no golden vectors or unit tests of its own (SURVEY.md §4), so this is the only pin there is.
"""
