"""CPU oracle for the passive-radar hot path -- TEST INFRASTRUCTURE ONLY.

Nothing under ``passiveradar_b200/`` may import this package.  The only
legitimate callers are ``tests/``, ``__graft_entry__.smoke()`` and the
``cpu_baseline`` / ``--impl reference`` legs of ``bench.py``, and there only as
the checker or the timed CPU baseline -- never as something the product path
falls back to.

What is in here
---------------
* ``xambg_oracle``    numpy/SciPy restatement of ``fast_xambg``
  (reference ``passiveRadar/range_doppler_processing.py:12-90``) with the same
  rounding points as the reference, plus a float64 "truth" from the closed
  form in SURVEY.md section 3.2.
* ``clutter_oracle``  restatements of ``LS_Filter``
  (``passiveRadar/clutter_removal.py:6-56``) and ``NLMS_filter``
  (``:189-249``), the definition of ``block_NLMS`` (absent from the reference;
  block length 1 is pinned to ``NLMS_filter``), and float64 truths.
* ``nlms_oracle.c``   the same NLMS recurrence in plain C (complex float
  arithmetic) so the 2M-sample BASELINE config can be checked in seconds; built
  by ``oracle/build.py`` into ``oracle/_build/`` (git-ignored).

How it is pinned
----------------
The reference is pure Python and imports in the build container, so the goldens
under ``tests/golden/`` were produced by *executing the reference's own
functions* (``tests/golden/make_golden.py``, run with the reference checkout on the
path) on the seeded inputs of ``passiveradar_b200.synth``.  ``tests/test_oracle_golden.py``
checks every function here against those files, so "oracle == reference" is a
tested statement, not an assumption.  The reference itself has no tests,
fixtures or golden vectors of its own (SURVEY.md section 4).
"""
