"""CPU oracle for the allRank scoring + listwise-loss + metric hot path.

TEST INFRASTRUCTURE ONLY.  Nothing under ``oracle/`` is part of the product:
only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` /
``--impl reference`` legs may import it, and only as the checker (or, for the
bench, as the timed CPU arm).  ``allrank_b200`` never imports this package and
fails loudly when its CUDA library is missing.

What is here
------------
* ``metrics_ref``  -- dcg / ndcg / mrr          (reference: allrank/models/metrics.py)
* ``losses_ref``   -- listNet, listMLE, approxNDCGLoss, lambdaLoss (7 weighing
                      schemes), neuralNDCG (+ NeuralSort, Sinkhorn)
                                               (reference: allrank/models/losses/*.py)
* ``scorer_ref``   -- LTRModel forward: FC -> pre-norm Transformer encoder -> head
                                               (reference: allrank/models/{model,transformer}.py)

Each function is a *restatement* in plain eager PyTorch on CPU tensors (fp32 by
default, fp64 on request), written from the algorithm, not copied; every
function cites the reference file:line it follows.

Pinning
-------
The reference is pure Python and importable wherever an allRank source tree is available (behind the
three stub modules in ``oracle/_stubs``).  ``oracle/make_golden.py`` imports the
*unmodified* reference from ``/root/reference``, runs it on seeded inputs and
commits the input/output vectors under ``tests/golden/``; ``tests/test_oracle_*``
check this restatement against (a) every known-answer value the reference's own
tests hold for the path (SURVEY.md section 8c) and (b) those golden vectors.
The encoder has no test in the reference; it is pinned only by the golden
vectors generated from the reference's ``make_model``.
"""
