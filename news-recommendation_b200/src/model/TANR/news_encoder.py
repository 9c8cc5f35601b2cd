"""TANR NewsEncoder (replaces reference src/model/TANR/news_encoder.py:9-54): title CNN + additive pooling."""
import torch.nn as nn

from model.general.attention.additive import AdditiveAttention
from model.general.cnn_text import BadIdFlag, cnn_text_encode, make_title_cnn
from newsrec_b200 import require_cuda
from newsrec_b200.ops import OperandCache


class NewsEncoder(nn.Module):
    def __init__(self, config, pretrained_word_embedding):
        super().__init__()
        self.config = config
        if pretrained_word_embedding is None:
            self.word_embedding = nn.Embedding(config.num_words, config.word_embedding_dim, padding_idx=0)
        else:
            self.word_embedding = nn.Embedding.from_pretrained(pretrained_word_embedding, freeze=False, padding_idx=0)
        self.title_CNN = make_title_cnn(config.num_filters, config.window_size, config.word_embedding_dim)
        self.title_attention = AdditiveAttention(config.query_vector_dim, config.num_filters)
        self._cache, self._flag = OperandCache(), BadIdFlag()

    def encode_ids(self, title):
        p = self.config.dropout_probability if self.training else 0.0
        return cnn_text_encode(title, self.word_embedding, self.title_CNN, self.title_attention, p, self._cache, "title", self._flag)

    def forward(self, news):
        dev = require_cuda()
        return self.encode_ids(news["title"].to(dev, non_blocking=True))
