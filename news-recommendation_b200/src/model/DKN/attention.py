"""Parameter container of the DKN history attention (reference src/model/DKN/attention.py:6-18): Linear(2F', 16), Linear(16, 1).
With no nonlinearity between the two Linears the score of history row h_j is alpha.c + beta.h_j + const; the softmax over j
cancels alpha.c + const, so the user vector does not depend on the candidate (DESIGN.md section 3, nr_dkn_user_*)."""
import torch
import torch.nn as nn


class Attention(torch.nn.Module):
    def __init__(self, config):
        super().__init__()
        self.config = config
        self.dnn = nn.Sequential(nn.Linear(len(config.window_sizes) * 2 * config.num_filters, 16), nn.Linear(16, 1))

    def weights(self):
        """(W1 (16, 2F'), b1, w2 (1, 16), b2)"""
        return self.dnn[0].weight, self.dnn[0].bias, self.dnn[1].weight, self.dnn[1].bias
