"""CPU oracle for Hi-Fi Ark (reference src/model/HiFiArk/**, general/attention/self.py, general/attention/similarity.py,
general/click_predictor/DNN.py), on top of newsrec_oracle's CNN text encoder.  TEST INFRASTRUCTURE ONLY, like
newsrec_oracle.py.  Pinned against tests/golden/hifiark.npz (oracle/make_golden_hifiark.py).

The kernels run everything after the news encoder in fp32 from fp32 news vectors and fp32 weights, so the storage contract
only touches the news encoder (newsrec_oracle.Contract).  `user_c` rounds the user side's inputs for the precision study.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

import newsrec_oracle as O


def hifiark_shapes(V, d=300, q=200, Fn=300, window=3, heads=5):
    s = {"news_encoder.word_embedding.weight": (V, d),
         "news_encoder.title_CNN.weight": (Fn, 1, window, d), "news_encoder.title_CNN.bias": (Fn,),
         "news_encoder.abstract_CNN.weight": (Fn, 1, window, d), "news_encoder.abstract_CNN.bias": (Fn,)}
    s.update(O._additive_shapes("news_encoder.title_attention", q, Fn))
    hid = int(math.sqrt(2 * Fn))
    s.update({"omap.W": (Fn, heads), "click_predictor.dnn.0.weight": (hid, 2 * Fn), "click_predictor.dnn.0.bias": (hid,),
              "click_predictor.dnn.2.weight": (1, hid), "click_predictor.dnn.2.bias": (1,)})
    return s


def hifiark_state_dict(V, seed):
    # the reference initialises W uniform(-0.1, 0.1) (OMAP.py:12-14)
    return O.det_state_dict(hifiark_shapes(V), seed, {"omap.W": 0.1})


def user_archive(x, W):
    """self.py:13-25 + residual (__init__.py:55-58) + OMAP.py:16-35 without the regulariser.  x (B, H, F) -> (B, P, F)."""
    y = torch.bmm(F.softmax(torch.bmm(x, x.transpose(1, 2)), dim=2), x) + x
    w = F.softmax(torch.matmul(y, W).transpose(1, 2), dim=2)
    return torch.bmm(w, y)


def regularizer(W):
    """OMAP.py:36-44."""
    P = W.shape[1]
    return (torch.mm(W.t(), W) * (1 - torch.eye(P, dtype=W.dtype))).norm(p="fro")


def score(cand, archive, p):
    """similarity.py:12-29 + DNN.py:19-28.  cand (n, F), archive (n, P, F) -> (n,)."""
    w = F.softmax(torch.bmm(archive, cand.unsqueeze(2)).squeeze(2), dim=1)
    u = torch.bmm(w.unsqueeze(1), archive).squeeze(1)
    h = F.relu(F.linear(torch.cat((cand, u), dim=1), p["click_predictor.dnn.0.weight"], p["click_predictor.dnn.0.bias"]))
    return F.linear(h, p["click_predictor.dnn.2.weight"], p["click_predictor.dnn.2.bias"]).squeeze(1)


def hifiark_forward(cand_title, clicked_title, p, c: O.Contract = O.EXACT, drop=None, user_c: O.Contract = O.EXACT,
                    with_reg=False):
    """__init__.py:22-65.  cand_title (B, C, T), clicked_title (B, H, T).  Returns (logits (B, C), regulariser or None,
    cand vectors, clicked vectors, archive).  drop: see newsrec_oracle.cnn_text_encoder (browsed block first, as packed)."""
    B, C, T = cand_title.shape
    H = clicked_title.shape[1]
    d_h = None if drop is None else dict(drop, n0=0)
    d_c = None if drop is None else dict(drop, n0=B * H)
    cv = O.tanr_news_encoder(cand_title.reshape(B * C, T), p, c, drop=d_c).view(B, C, -1)
    hv = O.tanr_news_encoder(clicked_title.reshape(B * H, T), p, c, drop=d_h).view(B, H, -1)
    q = {k: user_c.operand(v) for k, v in p.items() if not k.startswith("news_encoder.")}
    archive = user_archive(user_c.operand(hv), q["omap.W"])
    Fn = cv.shape[-1]
    logits = score(user_c.operand(cv).reshape(B * C, Fn), archive.repeat_interleave(C, dim=0), q).view(B, C)
    reg = regularizer(q["omap.W"]) if with_reg else None
    return logits, reg, cv, hv, archive


def get_prediction(cand, archive, p):
    """__init__.py:95-111: one candidate (F,) against one archive (P, F) -> 0-dim."""
    return score(cand.unsqueeze(0), archive.unsqueeze(0), p).squeeze(0)
