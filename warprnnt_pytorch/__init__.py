"""Top-level alias so that the reference's ``from warprnnt_pytorch import RNNTLoss``
(rnnt/models.py:8-11, cli/lightning.py:12) resolves to the H100 implementation when this
repository is on PYTHONPATH.  See INTEGRATION.md."""
from edgedict_b200.warprnnt_pytorch import RNNTLoss, rnnt_loss, certify_inputs  # noqa: F401

__all__ = ['rnnt_loss', 'RNNTLoss']
