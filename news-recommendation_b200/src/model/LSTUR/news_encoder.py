"""LSTUR NewsEncoder (replaces reference src/model/LSTUR/news_encoder.py:9-76):
[category embedding | subcategory embedding | title CNN + additive pooling] -> (batch, 3 * num_filters)."""
import torch
import torch.nn as nn

from model.general.attention.additive import AdditiveAttention
from model.general.cnn_text import BadIdFlag, cnn_text_encode, make_title_cnn
from newsrec_b200 import require_cuda
from newsrec_b200.ops import OperandCache
from newsrec_b200.ops_cnn import EmbeddingF32Fn


class NewsEncoder(nn.Module):
    def __init__(self, config, pretrained_word_embedding):
        super().__init__()
        self.config = config
        if pretrained_word_embedding is None:
            self.word_embedding = nn.Embedding(config.num_words, config.word_embedding_dim, padding_idx=0)
        else:
            self.word_embedding = nn.Embedding.from_pretrained(pretrained_word_embedding, freeze=False, padding_idx=0)
        self.category_embedding = nn.Embedding(config.num_categories, config.num_filters, padding_idx=0)
        self.title_CNN = make_title_cnn(config.num_filters, config.window_size, config.word_embedding_dim)
        self.title_attention = AdditiveAttention(config.query_vector_dim, config.num_filters)
        self._cache, self._flag, self._cat_flag = OperandCache(), BadIdFlag(), BadIdFlag()

    def encode(self, fields):
        """fields: category (n,), subcategory (n,), title (n, T) device int64 -> (n, 3F)"""
        dev = require_cuda()
        cat = EmbeddingF32Fn.apply(fields["category"], self.category_embedding.weight, self._cat_flag.get(dev))
        sub = EmbeddingF32Fn.apply(fields["subcategory"], self.category_embedding.weight, self._cat_flag.get(dev))
        p = self.config.dropout_probability if self.training else 0.0
        title = cnn_text_encode(fields["title"], self.word_embedding, self.title_CNN, self.title_attention, p, self._cache,
                                "title", self._flag, accurate=getattr(self.config, "precision", "fast") == "accurate")
        return torch.cat([cat, sub, title], dim=1)

    def forward(self, news):
        dev = require_cuda()
        return self.encode({k: news[k].to(dev, non_blocking=True) for k in ("category", "subcategory", "title")})
