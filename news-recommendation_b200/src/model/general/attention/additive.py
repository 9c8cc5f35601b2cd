"""AdditiveAttention on the fused wgmma pooling kernel (replaces reference
src/model/general/attention/additive.py:6-53; same constructor, parameter names and shapes)."""
import torch
import torch.nn as nn

from newsrec_b200.ops import AdditiveAttentionFn, OperandCache


class AdditiveAttention(nn.Module):
    def __init__(self, query_vector_dim, candidate_vector_dim, writer=None, tag=None, names=None):
        super().__init__()
        self.linear = nn.Linear(candidate_vector_dim, query_vector_dim)
        self.attention_query_vector = nn.Parameter(torch.empty(query_vector_dim).uniform_(-0.1, 0.1))
        # the reference's TensorBoard hook is accepted for signature compatibility; no caller enables it
        self.writer, self.tag, self.names = writer, tag, names
        self._cache = OperandCache()

    def forward(self, candidate_vector):
        """(batch, candidate_size, dim) -> (batch, dim)"""
        return AdditiveAttentionFn.apply(candidate_vector, self.linear.weight, self.linear.bias,
                                         self.attention_query_vector, self._cache, "additive")
