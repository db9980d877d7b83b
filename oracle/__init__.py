"""CPU oracle for the Competitive-Collaboration hot path.

TEST INFRASTRUCTURE ONLY.  Nothing under ``cc_b200/`` may import this package;
only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline /
``--impl reference`` legs do.  It is a plain-PyTorch fp32 restatement of the
reference's algorithm (anuragranj/cc @ 2b4e362); every function cites the
reference file:line it follows.

Parity pinning: the reference ships NO golden vectors or unit tests
(SURVEY.md section 4), so the oracle is pinned against *outputs of the reference
itself* - ``tests/golden/make_golden.py`` imports
a checkout of the reference (``$CC_REFERENCE``) and freezes its outputs (and autograd gradients) into
``tests/golden/*.npz``; ``tests/test_oracle_golden.py`` checks this package
against those fixtures.  The third-party ``spatial_correlation_sampler`` used by
Back2Future is absent from the tree: that one boundary is "parity unpinned"
(see ``oracle/nets.py``).
"""
from . import geometry, ssim, losses, nets, step  # noqa: F401
