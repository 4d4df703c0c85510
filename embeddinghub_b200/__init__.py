"""embeddinghub_b200 — H100-native ANN search backend for embeddinghub.

Only the k-NN hot path of featureform/embeddinghub is implemented here (see
DESIGN.md): a hand-written sm_90a CUDA library behind a C ABI
(include/ehb200.h) plus the host-side mirrors of the reference's interfaces for
that path.
"""
from ._native import EhbError, NativeIndex, NO_LABEL, ShardedIndex, lib  # noqa: F401
from .ann_index import ANNIndex  # noqa: F401
from .hub import EmbeddingHub, HubError  # noqa: F401
from . import offline  # noqa: F401

__all__ = ["ANNIndex", "EmbeddingHub", "HubError", "NativeIndex", "ShardedIndex", "EhbError", "NO_LABEL", "lib", "offline"]
