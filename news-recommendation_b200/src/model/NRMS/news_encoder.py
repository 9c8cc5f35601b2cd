"""NRMS NewsEncoder: embedding gather -> dropout -> MHSA -> dropout -> additive pooling, fused on sm_90a
(replaces reference src/model/NRMS/news_encoder.py:10-48; same submodule / parameter names)."""
import torch
import torch.nn as nn

from model.general.attention.additive import AdditiveAttention
from model.general.attention.multihead_self import MultiHeadSelfAttention
from newsrec_b200 import require_cuda
from newsrec_b200.guard import BadIdFlag
from newsrec_b200.ops import MhsaPoolEncoderFn, OperandCache, precision_mode


class NewsEncoder(nn.Module):
    def __init__(self, config, pretrained_word_embedding):
        super().__init__()
        self.config = config
        if pretrained_word_embedding is None:
            self.word_embedding = nn.Embedding(config.num_words, config.word_embedding_dim, padding_idx=0)
        else:
            self.word_embedding = nn.Embedding.from_pretrained(pretrained_word_embedding, freeze=False, padding_idx=0)
        self.multihead_self_attention = MultiHeadSelfAttention(config.word_embedding_dim, config.num_attention_heads)
        self.additive_attention = AdditiveAttention(config.query_vector_dim, config.word_embedding_dim)
        self._cache = OperandCache()
        self._flag = BadIdFlag()

    def bad_id_flag(self, dev):
        """Device int the gather sets for an id outside [0, num_words); polled without a sync on every call (guard.py)."""
        return self._flag.get(dev)

    def encode_ids(self, ids):
        """ids: int64 (n_titles, num_words_title) on the device -> (n_titles, word_embedding_dim)."""
        dev = require_cuda()
        a = self.additive_attention
        p = self.config.dropout_probability if self.training else 0.0
        return MhsaPoolEncoderFn.apply(ids, None, self.word_embedding.weight,
                                       *self.multihead_self_attention.qkv_parameters(),
                                       a.linear.weight, a.linear.bias, a.attention_query_vector,
                                       self.config.num_attention_heads, p, self._cache, "news", self.bad_id_flag(dev),
                                       precision_mode(self.config))

    def forward(self, news):
        """news: {"title": (batch, num_words_title) int64} -> (batch, word_embedding_dim)"""
        dev = require_cuda()
        return self.encode_ids(news["title"].to(dev, non_blocking=True))
