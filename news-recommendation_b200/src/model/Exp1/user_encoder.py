"""Exp1 UserEncoder (replaces reference src/model/Exp1/user_encoder.py:7-30): NRMS's user encoder on the browsed-news vectors
plus a learned position embedding.  The addend is applied inside the kernels' input conversion (fp32 sum, one rounding) and
its gradient is reduced on the device."""
import torch
import torch.nn as nn

from model.general.attention.additive import AdditiveAttention
from model.general.attention.multihead_self import MultiHeadSelfAttention
from newsrec_b200 import NewsrecError
from newsrec_b200.ops import MhsaPoolEncoderFn, OperandCache, precision_mode


class UserEncoder(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.config = config
        self.multihead_self_attention = MultiHeadSelfAttention(config.word_embedding_dim, config.num_attention_heads)
        self.position_embedding = nn.Parameter(
            torch.empty(config.num_clicked_news_a_user, config.word_embedding_dim).uniform_(-0.1, 0.1))
        self.additive_attention = AdditiveAttention(config.query_vector_dim, config.word_embedding_dim)
        self._cache = OperandCache()

    def forward(self, user_vector):
        """(batch, num_clicked_news_a_user, dim) fp32, any strides -> (batch, dim)"""
        if user_vector.dim() != 3 or user_vector.shape[1:] != self.position_embedding.shape:
            raise NewsrecError(f"Exp1 user encoder: browsed-news vectors of shape {tuple(user_vector.shape)}, the position embedding "
                               f"needs (batch, {self.position_embedding.shape[0]}, {self.position_embedding.shape[1]}) "
                               "(num_clicked_news_a_user)")
        a = self.additive_attention
        return MhsaPoolEncoderFn.apply(None, user_vector, None, *self.multihead_self_attention.qkv_parameters(),
                                       a.linear.weight, a.linear.bias, a.attention_query_vector,
                                       self.config.num_attention_heads, 0.0, self._cache, "user", None,
                                       precision_mode(self.config), self.position_embedding)
