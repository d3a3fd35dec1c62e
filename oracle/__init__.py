"""CPU oracle for the FullSubNet+/FullSubNet inference forward.

TEST INFRASTRUCTURE ONLY.  Nothing under ``oracle/`` is on the product path:
only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline /
``--impl reference`` legs may import it, and there only as the checker.

Parity status: PINNED.  ``oracle/fsn_oracle.py`` is checked against outputs of
the unmodified reference (imported read-only from a checkout of it by
``tests/golden/make_golden.py``; the resulting vectors are committed under
``tests/golden/``).  The reference itself ships no tests or golden vectors
(SURVEY.md section 4), so these generated fixtures are the pin.
"""
