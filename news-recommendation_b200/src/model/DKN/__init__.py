"""DKN drop-in (replaces reference src/model/DKN/__init__.py:7-104, KCNN.py, attention.py and general/click_predictor/DNN.py).
The news encoder is one kernel pair each way (nr_kcnn_encoder_*); after it, the history attention gives ONE user vector per
user (nr_dkn_user_*) and the DNN click predictor runs as the archive scorer with a one-row archive, which evaluation also uses."""
import torch

from model.DKN.KCNN import KCNN
from model.DKN.attention import Attention
from model.HiFiArk import DNNClickPredictor
from newsrec_b200 import NewsrecError, require_cuda
from newsrec_b200.ops_dkn import DknStepFn, DknUserFn, dkn_score, score_impressions
from newsrec_b200.pack import SlotPacker


class DKN(torch.nn.Module):
    def __init__(self, config, pretrained_word_embedding=None, pretrained_entity_embedding=None, pretrained_context_embedding=None):
        super().__init__()
        self.config = config
        self.kcnn = KCNN(config, pretrained_word_embedding, pretrained_entity_embedding, pretrained_context_embedding)
        self.attention = Attention(config)
        self.click_predictor = DNNClickPredictor(len(config.window_sizes) * 2 * config.num_filters)
        self._title_packer, self._entity_packer = SlotPacker(), SlotPacker()

    def _widths(self):
        return self.config.num_filters, len(self.config.window_sizes)

    def forward(self, candidate_news, clicked_news):
        """-> click logits (batch, 1 + K)"""
        dev = require_cuda()
        C, H = len(candidate_news), len(clicked_news)
        title, B = self._title_packer.pack(clicked_news, candidate_news, "title", dev)
        entities, _ = self._entity_packer.pack(clicked_news, candidate_news, "title_entities", dev)
        vec = self.kcnn.encode_ids(title, entities)  # B*H history rows, then B*C candidate rows
        return DknStepFn.apply(vec, B, H, C, *self._widths(), *self.attention.weights(), *self.click_predictor.weights())

    def get_news_vector(self, news):
        """-> (batch, len(window_sizes) * num_filters)"""
        return self.kcnn(news)

    def get_user_vector(self, clicked_news_vector):
        """(batch, H, len(window_sizes) * num_filters) -> the same, as the reference"""
        return clicked_news_vector

    def pool_user_vector(self, clicked_news_vector):
        """(batch, H, F') -> (batch, F'): the one attention vector per user that the click predictor scores against, the user
        operand of the whole-pool kernels (newsrec_b200.recommend, pool_eval)"""
        require_cuda()
        W1a, _, w2a, _ = self.attention.weights()
        return DknUserFn.apply(clicked_news_vector, W1a, w2a)

    def get_prediction(self, candidate_news_vector, clicked_news_vector):
        """candidates (n, F'), clicked (H, F') -> click logits (n,)"""
        dev = require_cuda()
        if candidate_news_vector.dim() != 2 or clicked_news_vector.dim() != 2:
            raise NewsrecError(f"get_prediction: candidates {tuple(candidate_news_vector.shape)} against clicked news "
                               f"{tuple(clicked_news_vector.shape)}; expected (n, F) and (H, F)")
        W1a, _, w2a, _ = self.attention.weights()
        user = DknUserFn.apply(clicked_news_vector.to(dev).unsqueeze(0), W1a, w2a)
        return dkn_score(candidate_news_vector.to(dev), user[0], *self._widths(), *self.click_predictor.weights())

    def score_impressions(self, news_matrix, cand_index, seg_offsets, clicked, bad_flag):
        """Device evaluation (newsrec_b200.evaluate): clicked (S, H, F') the history rows of each impression's user."""
        W1a, _, w2a, _ = self.attention.weights()
        return score_impressions(news_matrix, cand_index, seg_offsets, clicked, *self._widths(), W1a, w2a,
                                 *self.click_predictor.weights(), bad_flag)
