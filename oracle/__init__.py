"""CPU oracle for the UnionML batch-predict hot path.  TEST INFRASTRUCTURE ONLY.

This package restates, on the CPU, the algorithm the reference runs for
``dataset.reader / feature_loader -> Model.predict -> @model.predictor`` with the canonical
``LogisticRegression`` predictor.  It exists to *check* the CUDA path; it is never the product:

* only ``tests/``, ``__graft_entry__.smoke()`` and the ``cpu_baseline`` / ``--impl reference``
  legs of ``bench.py`` may import or execute anything under ``oracle/``;
* nothing under ``unionml_b200/`` imports it, and the product path raises when the CUDA
  library is missing instead of falling back to this code.

Where the arithmetic lives: UnionML itself contains none.  The user predictor
(``unionml:README.md:87-92``) calls scikit-learn's
``LinearClassifierMixin.predict`` (``sklearn/linear_model/_base.py:366-427``, scikit-learn is
*unpinned* in ``unionml:requirements.txt:12``; 1.9.0 is what the fixtures were made with), which is
``X @ coef_.T + intercept_ -> argmax(axis=1) -> classes_.take``.  ``oracle.linear`` restates that
published algorithm in numpy and ``oracle/linear_predict.c`` in plain C (``oracle.c_port`` loads it); ``oracle.unionml_path`` restates the UnionML wrapper around it
(no flytekit); ``oracle.mlp`` restates the PyTorch quickstart predictor.

Parity pinning (see ``tests/test_oracle_golden.py``): the restatement is checked against
(1) the only numeric known-answer in the reference's tests,
``unionml:tests/unit/test_aws_lambda_handler.py:117-127,134-159`` -> ``[8.0, 8.0, 0.0]``,
(2) the quickstart sample ``[6, 9, 3, 7, 2]``, and (3) scikit-learn itself, run in-process, on
seeded batches (scikit-learn *is* the reference's arithmetic and is importable here and on the
GPU box).  Fixtures and their generator are committed under ``tests/golden/``.
"""
