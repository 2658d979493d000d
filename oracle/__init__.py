"""oracle/ -- TEST INFRASTRUCTURE ONLY.

CPU restatement (torch fp32/fp64 on the host) of the structured-distillation
step of irfanICMLL/structure_knowledge_distillation, plus the recipe that
compiles the reference's own `libs/src/bn.cu` into `oracle/_ref/`.

Nothing under `structure_knowledge_distillation_b200/` may import this package.
Only `tests/`, `__graft_entry__.smoke()` and the `cpu_baseline` / `--impl
reference` legs of `bench.py` use it, and only as the checker or as the
timed CPU baseline -- never as part of the product path.

Parity pinning: the reference ships no tests / golden vectors (SURVEY.md §4).
`oracle/port.py` is therefore pinned by differential execution against the
reference's own Python modules imported from a checkout of it
(`oracle/refshim.py`, `oracle/make_golden.py`) -- the resulting fixtures are
committed under `tests/golden/` and re-checked by `tests/test_oracle_golden.py`.
"""
