"""Exp1 NewsEncoder (replaces reference src/model/Exp1/news_encoder.py:10-110): the NRMS title encoder and NAML's category /
subcategory element encoders (one shared category table), fused by additive attention.  Same submodule / parameter names.

precision "accurate" (config.precision, DESIGN.md section 4): the title view is NRMS's accurate news encoder and the stacked
views enter final_attention as hi/lo bf16 pairs -- the history-level MHSA of the user encoder amplifies a plain bf16 rounding
there to 2-3e-3 of the logits."""
import torch
import torch.nn as nn

from model.general.attention.additive import AdditiveAttention
from model.general.attention.multihead_self import MultiHeadSelfAttention
from model.NAML.news_encoder import ElementEncoder
from newsrec_b200 import NewsrecError, require_cuda
from newsrec_b200.guard import BadIdFlag
from newsrec_b200.ops import AdditiveAttentionFn, MhsaPoolEncoderFn, OperandCache, precision_mode


class TextEncoder(nn.Module):
    def __init__(self, word_embedding, word_embedding_dim, num_attention_heads, query_vector_dim, dropout_probability):
        super().__init__()
        self.word_embedding = word_embedding
        self.dropout_probability = dropout_probability
        self.multihead_self_attention = MultiHeadSelfAttention(word_embedding_dim, num_attention_heads)
        self.additive_attention = AdditiveAttention(query_vector_dim, word_embedding_dim)
        self._cache, self._flag = OperandCache(), BadIdFlag()

    def forward(self, text, precision="fast"):
        """(batch, num_words) int64 on the device -> (batch, word_embedding_dim)"""
        dev = require_cuda()
        a, mhsa = self.additive_attention, self.multihead_self_attention
        p = self.dropout_probability if self.training else 0.0
        return MhsaPoolEncoderFn.apply(text, None, self.word_embedding.weight, *mhsa.qkv_parameters(),
                                       a.linear.weight, a.linear.bias, a.attention_query_vector,
                                       mhsa.num_attention_heads, p, self._cache, "news", self._flag.get(dev), precision)


class NewsEncoder(nn.Module):
    TEXT, ELEMENT = ("title",), ("category", "subcategory")

    def __init__(self, config, pretrained_word_embedding):
        super().__init__()
        self.config = config
        attrs = config.dataset_attributes["news"]
        assert len(attrs) > 0
        if "abstract" in attrs:
            raise NewsrecError("Exp1 with an 'abstract' view is not supported (the reference leaves it as a TODO); configure "
                               "dataset_attributes['news'] from 'title', 'category', 'subcategory'")
        if pretrained_word_embedding is None:
            word_embedding = nn.Embedding(config.num_words, config.word_embedding_dim, padding_idx=0)
        else:
            word_embedding = nn.Embedding.from_pretrained(pretrained_word_embedding, freeze=False, padding_idx=0)
        self.text_encoders = nn.ModuleDict({
            name: TextEncoder(word_embedding, config.word_embedding_dim, config.num_attention_heads, config.query_vector_dim,
                              config.dropout_probability)
            for name in self.TEXT if name in attrs})
        category_embedding = nn.Embedding(config.num_categories, config.category_embedding_dim, padding_idx=0)
        self.element_encoders = nn.ModuleDict({
            name: ElementEncoder(category_embedding, config.category_embedding_dim, config.word_embedding_dim)
            for name in self.ELEMENT if name in attrs})
        if len(attrs) > 1:
            self.final_attention = AdditiveAttention(config.query_vector_dim, config.word_embedding_dim)

    def names(self):
        return list(self.text_encoders.keys()) + list(self.element_encoders.keys())

    def encode(self, fields):
        """fields: name -> device tensor ((n, T) for the title, (n,) for elements) -> (n, word_embedding_dim)"""
        mode = precision_mode(self.config)
        vectors = [enc(fields[name], mode) for name, enc in self.text_encoders.items()]
        vectors += [enc(fields[name]) for name, enc in self.element_encoders.items()]
        if len(vectors) == 1:
            return vectors[0]
        fa = self.final_attention
        return AdditiveAttentionFn.apply(torch.stack(vectors, dim=1), fa.linear.weight, fa.linear.bias, fa.attention_query_vector,
                                         fa._cache, "additive", mode)

    def forward(self, news):
        """news: {"category", "subcategory": (batch,), "title": (batch, num_words_title)} -> (batch, word_embedding_dim)"""
        dev = require_cuda()
        return self.encode({k: news[k].to(dev, non_blocking=True) for k in self.names()})
