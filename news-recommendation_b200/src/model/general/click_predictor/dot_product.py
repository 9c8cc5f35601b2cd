"""DotProductClickPredictor on the sm_90a dot-score kernel (replaces reference
src/model/general/click_predictor/dot_product.py:4-19; same class name and call signature)."""
import torch

from newsrec_b200.ops import DotScoreFn


class DotProductClickPredictor(torch.nn.Module):
    def forward(self, candidate_news_vector, user_vector):
        """(batch, candidates, X), (batch, X) -> (batch, candidates) raw logits."""
        return DotScoreFn.apply(candidate_news_vector, user_vector)
