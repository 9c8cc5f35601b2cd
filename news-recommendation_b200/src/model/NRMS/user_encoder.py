"""NRMS UserEncoder: MHSA over the browsed-news vectors -> additive pooling, fused on sm_90a
(replaces reference src/model/NRMS/user_encoder.py:6-26)."""
import torch.nn as nn

from model.general.attention.additive import AdditiveAttention
from model.general.attention.multihead_self import MultiHeadSelfAttention
from newsrec_b200.ops import MhsaPoolEncoderFn, OperandCache, precision_mode


class UserEncoder(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.config = config
        self.multihead_self_attention = MultiHeadSelfAttention(config.word_embedding_dim, config.num_attention_heads)
        self.additive_attention = AdditiveAttention(config.query_vector_dim, config.word_embedding_dim)
        self._cache = OperandCache()

    def forward(self, user_vector):
        """(batch, num_clicked_news_a_user, dim) fp32, any strides -> (batch, dim)"""
        a = self.additive_attention
        return MhsaPoolEncoderFn.apply(None, user_vector, None, *self.multihead_self_attention.qkv_parameters(),
                                       a.linear.weight, a.linear.bias, a.attention_query_vector,
                                       self.config.num_attention_heads, 0.0, self._cache, "user", None,
                                       precision_mode(self.config))  # precise mode: fp32-accurate forward
