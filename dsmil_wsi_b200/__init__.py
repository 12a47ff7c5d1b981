"""dsmil_wsi_b200 -- H100-native DSMIL aggregator hot path (see DESIGN.md).

Public surface == the reference's dsmil.py: FCLayer, IClassifier, BClassifier, MILNet.
"""
from .modules import BClassifier, FCLayer, IClassifier, MILNet  # noqa: F401

__all__ = ["FCLayer", "IClassifier", "BClassifier", "MILNet"]
