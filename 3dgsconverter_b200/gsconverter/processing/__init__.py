"""gsx drop-in for the reference's ``gsconverter.processing`` package.

Exports the same single name the reference exports (``DataProcessor``); ``gpu_ops`` is a sibling module
imported on demand by ``data_processor`` and by ``formats/sog.py``.  All keep-masks and the K-Means run on
libgsx.so (hand-written sm_90a CUDA); see INTEGRATION.md for the three ways to wire it in.
"""
from . import data_processor as _data_processor

DataProcessor = _data_processor.DataProcessor

__all__ = ("DataProcessor",)
