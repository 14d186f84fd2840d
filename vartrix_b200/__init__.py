"""vartrix_b200 -- H100-native engine for the per-locus read-scoring path of 10XGenomics/vartrix.

The product is the CUDA library behind include/vartrix_b200.h (csrc/); this package is its thin
Python host mirror.  Importing it does not need a GPU; creating an Engine does."""
from .engine import Barcodes, Engine, SlimBatch, StagedBatch, Triplets, VtxError, pack_cb, pack_umi, shard_bounds  # noqa: F401
from . import synth, mtx  # noqa: F401

__all__ = ["Barcodes", "Engine", "SlimBatch", "StagedBatch", "pack_cb", "Triplets", "VtxError", "pack_umi", "shard_bounds", "synth", "mtx"]
