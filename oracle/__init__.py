"""CPU oracle for the EsViT multi-crop self-distillation step.

TEST INFRASTRUCTURE ONLY.  Nothing under ``esvit_b200/`` may import this
package: it is the checker, never the product.  Only ``tests/``,
``__graft_entry__.smoke()`` and the ``cpu_baseline`` / ``--impl reference``
legs of ``bench.py`` may use it.

The oracle is a *functional* plain-PyTorch restatement (fp32, any device, CPU
by default) of the reference algorithm, operating directly on a reference
``state_dict``.  Every function cites the reference file:line it follows
(paths relative to the reference repository).

Pinning: the reference ships no tests, golden vectors or fixtures
(SURVEY.md §4), so the oracle is pinned against *outputs of the reference
itself run in the build container* — ``oracle/make_golden.py`` imports the
unmodified reference modules, runs them on seeded inputs and commits the
resulting vectors under ``tests/golden/``; ``tests/test_oracle_golden.py``
checks the oracle against them on every CPU run.
"""
