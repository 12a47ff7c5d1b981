"""Drop-in for the reference's `dsmil.py`: put this repo ahead of the reference on PYTHONPATH and
`import dsmil as mil` (train_tcga.py:224-225, train_mil.py:122-123, compute_feats.py:1,
attention_map.py:1) resolves here.  Same four classes, H100-native underneath."""
from dsmil_wsi_b200.modules import BClassifier, FCLayer, IClassifier, MILNet  # noqa: F401

__all__ = ["FCLayer", "IClassifier", "BClassifier", "MILNet"]
