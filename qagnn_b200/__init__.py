"""qagnn_b200 — H100-native (sm_90a) implementation of QA-GNN's graph-attention message-passing path.

Public surface mirrors the reference's modeling/modeling_qagnn.py:
    GATConvE, QAGNN_Message_Passing, QAGNN, LM_QAGNN, make_one_hot
"""
from .modeling_qagnn import GATConvE, QAGNN_Message_Passing, QAGNN, LM_QAGNN, make_one_hot  # noqa: F401

__all__ = ["GATConvE", "QAGNN_Message_Passing", "QAGNN", "LM_QAGNN", "make_one_hot"]
