"""CPU oracle for the SC-SfMLearner training hot path.  TEST INFRASTRUCTURE ONLY.

This package is a plain-PyTorch (CPU, fp32 or fp64) restatement of the reference
algorithm (JiawangBian/SC-SfMLearner-Release: inverse_warp.py, loss_functions.py,
models/*.py, train.py:249-282).  It is the *checker* for the CUDA kernels in
`sc-sfmlearner-release_b200/csrc/`.  Nothing in the product path may import it:
only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s CPU-baseline / `--impl
reference` leg do.

Parity status: PINNED.  The reference holds no golden vectors or tests of its own
(SURVEY.md section 4), so the oracle is pinned against the reference code itself:
`tests/golden/make_golden.py` imports the unmodified reference from a checkout of the
original project, runs it on seeded inputs and commits the input/output
vectors under `tests/golden/`; `tests/test_oracle_golden.py` checks every oracle
function against those vectors.  Third-party arithmetic the reference relies on
(`F.grid_sample`, `avg_pool2d`, `ReflectionPad2d`, torchvision ResNet, Adam: PyTorch
2.11.0 / torchvision 0.26.0, not vendored in the reference) is restated here
explicitly from its published definition, each function citing the call site.
"""
from . import geometry, losses  # noqa: F401
