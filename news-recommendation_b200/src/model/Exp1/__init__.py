"""Exp1 drop-in (replaces reference src/model/Exp1/__init__.py:7-84).  All 1+K+H news of a batch are packed per attribute
into one id tensor: one title-encoder call, one call per element view and one final-attention call for the whole batch.

Ensembles (reference train.py: ensemble_factor independent models, NLLLoss on the log of their mean softmax) are plain
torch around independent instances; each instance keeps its own operand caches."""
import torch

from model.Exp1.news_encoder import NewsEncoder
from model.Exp1.user_encoder import UserEncoder
from model.general.click_predictor.dot_product import DotProductClickPredictor
from newsrec_b200 import require_cuda
from newsrec_b200.pack import SlotPacker


class Exp1(torch.nn.Module):
    def __init__(self, config, pretrained_word_embedding=None):
        super().__init__()
        self.config = config
        self.news_encoder = NewsEncoder(config, pretrained_word_embedding)
        self.user_encoder = UserEncoder(config)
        self.click_predictor = DotProductClickPredictor()
        self._packer = SlotPacker()

    def forward(self, candidate_news, clicked_news):
        """lists of 1+K and num_clicked_news_a_user per-slot dicts {"category", "subcategory": (batch,), "title": (batch, T)}
        (slot-major, what the reference's DataLoader yields) -> (batch, 1+K) logits"""
        dev = require_cuda()
        C, H = len(candidate_news), len(clicked_news)
        fields, B = {}, None
        for name in self.news_encoder.names():  # (B*H + B*C, ...): browsed block, then candidates
            fields[name], B = self._packer.pack(clicked_news, candidate_news, name, dev)
        vec = self.news_encoder.encode(fields)
        d = vec.shape[1]
        user_vector = self.user_encoder(vec[:B * H].view(B, H, d))
        return self.click_predictor(vec[B * H:].view(B, C, d), user_vector)

    def get_news_vector(self, news):
        """{"category", "subcategory": (batch,), "title": (batch, T)} -> (batch, dim)"""
        return self.news_encoder(news)

    def get_user_vector(self, clicked_news_vector):
        """(batch, num_clicked_news_a_user, dim) -> (batch, dim)"""
        return self.user_encoder(clicked_news_vector)

    def get_prediction(self, news_vector, user_vector):
        """(candidates, dim), (dim,) -> (candidates,)"""
        return self.click_predictor(news_vector.unsqueeze(0), user_vector.unsqueeze(0)).squeeze(0)
