"""Hi-Fi Ark drop-in (replaces reference src/model/HiFiArk/__init__.py:9-111, OMAP.py, general/attention/self.py,
similarity.py and click_predictor/DNN.py).  After the news encoder, two kernels each way (csrc/archive.cu): the user side
(self-attention + residual + OMAP pooling into the archive, plus the orthogonality regulariser) and the similarity-attention
DNN scorer, which evaluation also uses."""
from math import sqrt

import torch
import torch.nn as nn

from model.HiFiArk.news_encoder import NewsEncoder
from newsrec_b200 import NewsrecError, require_cuda
from newsrec_b200.ops_hifiark import ArchiveScoreFn, ArchiveStepFn, ArchiveUserFn, score_impressions
from newsrec_b200.pack import SlotPacker


class OMAP(nn.Module):
    """Parameter container of the orthogonal multi-head pooling (reference HiFiArk/OMAP.py:8-14): W (num_filters, P)."""

    def __init__(self, config):
        super().__init__()
        self.config = config
        self.W = nn.Parameter(torch.empty(config.num_filters, config.num_pooling_heads).uniform_(-0.1, 0.1))


class DNNClickPredictor(nn.Module):
    """Parameter container of reference general/click_predictor/DNN.py:6-17: Linear(2F, int(sqrt(2F))), ReLU, Linear(., 1)."""

    def __init__(self, input_size, hidden_size=None):
        super().__init__()
        if hidden_size is None:
            hidden_size = int(sqrt(input_size))
        self.dnn = nn.Sequential(nn.Linear(input_size, hidden_size), nn.ReLU(), nn.Linear(hidden_size, 1))

    def weights(self):
        return self.dnn[0].weight, self.dnn[0].bias, self.dnn[2].weight, self.dnn[2].bias


class HiFiArk(torch.nn.Module):
    def __init__(self, config, pretrained_word_embedding=None):
        super().__init__()
        self.config = config
        self.news_encoder = NewsEncoder(config, pretrained_word_embedding)
        self.omap = OMAP(config)
        self.click_predictor = DNNClickPredictor(config.num_filters * 2)
        self._packer = SlotPacker()

    def forward(self, candidate_news, clicked_news):
        """-> (click logits (batch, 1+K), regularizer_loss: 0-dim in train mode, None in eval mode)"""
        dev = require_cuda()
        C, H = len(candidate_news), len(clicked_news)
        ids, B = self._packer.pack(clicked_news, candidate_news, "title", dev)
        vec = self.news_encoder.encode_ids(ids)  # B*H history rows, then B*C candidate rows
        logits, regularizer_loss = ArchiveStepFn.apply(vec, B, H, C, self.omap.W, *self.click_predictor.weights(), self.training)
        return logits, (regularizer_loss if self.training else None)

    def get_news_vector(self, news):
        """-> (batch, num_filters)"""
        return self.news_encoder(news)

    def get_user_vector(self, clicked_news_vector):
        """(batch, H, num_filters), any strides -> the archive (batch, num_pooling_heads, num_filters)"""
        require_cuda()
        return ArchiveUserFn.apply(clicked_news_vector, self.omap.W)

    def pool_user_vector(self, clicked_news_vector):
        """The user operand of the whole-pool kernels (newsrec_b200.recommend, pool_eval): the archive, as get_user_vector"""
        return self.get_user_vector(clicked_news_vector)

    def get_prediction(self, candidate_news_vector, user_archive_vector):
        """(num_filters,) -> 0-dim logit, as the reference; (n, num_filters) -> (n,), what the reference's evaluate.py passes.
        user_archive_vector: (num_pooling_heads, num_filters)."""
        dev = require_cuda()
        if candidate_news_vector.dim() not in (1, 2) or user_archive_vector.dim() != 2:
            raise NewsrecError(f"get_prediction: candidates {tuple(candidate_news_vector.shape)} against an archive "
                               f"{tuple(user_archive_vector.shape)}; expected (F,) or (n, F) and (P, F)")
        cand = candidate_news_vector.to(dev)
        rows = cand.unsqueeze(0) if cand.dim() == 1 else cand
        seg = torch.tensor([0, rows.shape[0]], dtype=torch.int64, device=dev)
        out = ArchiveScoreFn.apply(rows, seg, user_archive_vector.to(dev).unsqueeze(0), *self.click_predictor.weights())
        return out.squeeze(0) if cand.dim() == 1 else out

    def score_impressions(self, news_matrix, cand_index, seg_offsets, archives, bad_flag):
        """Device evaluation (newsrec_b200.evaluate): every impression against its user's archive, one launch."""
        return score_impressions(news_matrix, cand_index, seg_offsets, archives, *self.click_predictor.weights(), bad_flag)
