"""egnn_pytorch_b200 -- H100 (sm_90a) implementation of the EGNN hot path (forward and backward) behind the
reference's module API (`from egnn_pytorch import EGNN, EGNN_Network`, reference
egnn_pytorch/__init__.py:1)."""
from .egnn import EGNN, EGNN_Network, CoorsNorm, GlobalLinearAttention, edge_index_to_neighbors, radius_neighbors  # noqa: F401
from .egnn import radius_neighbors_wide, knn_neighbors  # noqa: F401
from .graphs import GraphedForward  # noqa: F401

__all__ = ["EGNN", "EGNN_Network"]
