"""DKN KCNN (replaces reference src/model/DKN/KCNN.py:9-117): word and transformed-entity channels, one Conv2d per window and
one additive attention shared by the windows, in one kernel pair each way (nr_kcnn_encoder_*).  Same parameters and names."""
import torch
import torch.nn as nn

from model.general.attention.additive import AdditiveAttention
from newsrec_b200 import NewsrecError, require_cuda
from newsrec_b200.guard import BadIdFlag
from newsrec_b200.ops import OperandCache
from newsrec_b200.ops_dkn import KcnnEncoderFn


class KCNN(torch.nn.Module):
    def __init__(self, config, pretrained_word_embedding, pretrained_entity_embedding, pretrained_context_embedding):
        super().__init__()
        self.config = config
        if config.use_context:  # the reference marks context embeddings as unavailable
            raise NewsrecError("DKN use_context=True: context embeddings are not supported (DESIGN.md section 6)")
        wins = list(config.window_sizes)
        if not 1 <= len(wins) <= 4 or not all(1 <= x <= 4 for x in wins):  # the reference takes any; the kernels 1 .. 4 of 1 .. 4
            raise NewsrecError(f"DKN window_sizes={wins}: the KCNN kernels take 1 to 4 windows of 1 to 4 words (include/newsrec_b200.h)")
        if pretrained_word_embedding is None:
            self.word_embedding = nn.Embedding(config.num_words, config.word_embedding_dim, padding_idx=0)
        else:
            self.word_embedding = nn.Embedding.from_pretrained(pretrained_word_embedding, freeze=False, padding_idx=0)
        if pretrained_entity_embedding is None:
            self.entity_embedding = nn.Embedding(config.num_entities, config.entity_embedding_dim, padding_idx=0)
        else:
            self.entity_embedding = nn.Embedding.from_pretrained(pretrained_entity_embedding, freeze=False, padding_idx=0)
        self.transform_matrix = nn.Parameter(
            torch.empty(config.entity_embedding_dim, config.word_embedding_dim).uniform_(-0.1, 0.1))
        self.transform_bias = nn.Parameter(torch.empty(config.word_embedding_dim).uniform_(-0.1, 0.1))
        self.conv_filters = nn.ModuleDict({
            str(x): nn.Conv2d(2, config.num_filters, (x, config.word_embedding_dim)) for x in config.window_sizes})
        self.additive_attention = AdditiveAttention(config.query_vector_dim, config.num_filters)
        self._cache, self._flag = OperandCache(), BadIdFlag()

    def encode_ids(self, title, entities):
        """title, entities: int64 (n, num_words_title) on the device -> (n, len(window_sizes) * num_filters)"""
        att = self.additive_attention
        convs = []
        for x in self.config.window_sizes:
            conv = self.conv_filters[str(x)]
            convs += [conv.weight, conv.bias]
        return KcnnEncoderFn.apply(title, entities, self._cache, "kcnn", self._flag.get(title.device), self.word_embedding.weight,
                                   self.entity_embedding.weight, self.transform_matrix, self.transform_bias, att.linear.weight,
                                   att.linear.bias, att.attention_query_vector, *convs)

    def forward(self, news):
        dev = require_cuda()
        return self.encode_ids(news["title"].to(dev, non_blocking=True), news["title_entities"].to(dev, non_blocking=True))
