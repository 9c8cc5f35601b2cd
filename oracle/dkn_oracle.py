"""CPU oracle for DKN (reference src/model/DKN/**, general/click_predictor/DNN.py).  TEST INFRASTRUCTURE ONLY, like
newsrec_oracle.py.  Pinned against tests/golden/dkn.npz (oracle/make_golden_dkn.py).

The windows are a list in the order of config.window_sizes, repeats kept: the reference runs one Conv2d per entry (a repeated
size runs the same conv twice) and concatenates the pooled vectors in that order.  The state_dict holds one conv per distinct
size, so the order cannot be read back from it.

Contract sites (newsrec_oracle.Contract) where the kernels store bf16: the word and entity rows and the transform matrix M
(operands), tanh(E M + b) (stored in the entity section of X2), the conv weights (operands), the conv output (stored), and the
attention weight Wa (operand).  Everything after the news encoder is fp32.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

import newsrec_oracle as O

WINDOWS = (2, 3, 4)


def dkn_shapes(V, VE, d=300, de=100, q=200, Fn=50, windows=WINDOWS):
    """One conv per distinct window size (the reference's ModuleDict); the DNN widths count every entry of `windows`."""
    s = {"kcnn.word_embedding.weight": (V, d), "kcnn.entity_embedding.weight": (VE, de),
         "kcnn.transform_matrix": (de, d), "kcnn.transform_bias": (d,)}
    for x in windows:
        s[f"kcnn.conv_filters.{x}.weight"] = (Fn, 2, x, d)
        s[f"kcnn.conv_filters.{x}.bias"] = (Fn,)
    s.update(O._additive_shapes("kcnn.additive_attention", q, Fn))
    Fp = len(windows) * Fn
    hid = int(math.sqrt(2 * Fp))
    s.update({"attention.dnn.0.weight": (16, 2 * Fp), "attention.dnn.0.bias": (16,), "attention.dnn.1.weight": (1, 16),
              "attention.dnn.1.bias": (1,), "click_predictor.dnn.0.weight": (hid, 2 * Fp), "click_predictor.dnn.0.bias": (hid,),
              "click_predictor.dnn.2.weight": (1, hid), "click_predictor.dnn.2.bias": (1,)})
    return s


def dkn_state_dict(V, VE, seed, **kw):
    # the reference initialises M and b uniform(-0.1, 0.1) (KCNN.py:41-45)
    return O.det_state_dict(dkn_shapes(V, VE, **kw), seed, {"kcnn.transform_matrix": 0.1, "kcnn.transform_bias": 0.1})


def synth_entities(titles, VE, seed):
    """title_entities of the same shape: mostly 0 (no entity), a few ids in [1, VE) with repeats, only on real tokens."""
    ids = O.det_randint(titles.shape, seed, 1, VE)
    keep = O.det_randint(titles.shape, seed + 1, 0, 4) == 0
    return ids * keep * (titles != 0)


def kcnn(title, entities, p, c: O.Contract = O.EXACT, windows=WINDOWS):
    """KCNN.py:56-117 (use_context=False).  title, entities (N, T) -> (N, len(windows) * F), window after window in the
    order of `windows`."""
    wv = O.embedding(title, p["kcnn.word_embedding.weight"], c)
    ev = O.embedding(entities, p["kcnn.entity_embedding.weight"], c)
    t = c.act(torch.tanh(torch.matmul(ev, c.operand(p["kcnn.transform_matrix"])) + p["kcnn.transform_bias"]))
    x2 = torch.stack([wv, t], dim=1)
    pooled = []
    for x in windows:
        y = F.conv2d(x2, c.operand(p[f"kcnn.conv_filters.{x}.weight"]), p[f"kcnn.conv_filters.{x}.bias"]).squeeze(3)
        y = c.act(F.relu(y).transpose(1, 2))
        pooled.append(O.additive_attention(y, p, "kcnn.additive_attention", c))
    return torch.cat(pooled, dim=1)


def attention_per_candidate(cand, hv, p):
    """attention.py:20-39 as the reference computes it, once per candidate.  cand (B, C, F'), hv (B, H, F') -> (B, C, F')."""
    B, C, Fp = cand.shape
    H = hv.shape[1]
    z = torch.cat([cand.unsqueeze(2).expand(B, C, H, Fp), hv.unsqueeze(1).expand(B, C, H, Fp)], dim=3)
    s = F.linear(F.linear(z, p["attention.dnn.0.weight"], p["attention.dnn.0.bias"]), p["attention.dnn.1.weight"],
                 p["attention.dnn.1.bias"]).squeeze(3)
    return torch.matmul(F.softmax(s, dim=2), hv)


def user_vector(hv, p):
    """The collapsed form the kernels compute: softmax_j(beta . h_j) with beta = W1[:, F':]^T w2.  hv (B, H, F') -> (B, F')."""
    Fp = hv.shape[2]
    beta = torch.matmul(p["attention.dnn.1.weight"].view(-1), p["attention.dnn.0.weight"][:, Fp:])
    w = F.softmax(torch.matmul(hv, beta), dim=1)
    return torch.bmm(w.unsqueeze(1), hv).squeeze(1)


def score(cand, user, p):
    """DNN.py:19-28: cand (n, F'), user (n, F') -> (n,)."""
    h = F.relu(F.linear(torch.cat((cand, user), dim=1), p["click_predictor.dnn.0.weight"], p["click_predictor.dnn.0.bias"]))
    return F.linear(h, p["click_predictor.dnn.2.weight"], p["click_predictor.dnn.2.bias"]).squeeze(1)


def dkn_forward(cand_title, cand_ent, clicked_title, clicked_ent, p, c: O.Contract = O.EXACT, windows=WINDOWS):
    """__init__.py:26-64.  (B, C, T) / (B, H, T) id tensors -> (logits (B, C), cand vectors, clicked vectors, user (B, F'))."""
    B, C, T = cand_title.shape
    H = clicked_title.shape[1]
    cv = kcnn(cand_title.reshape(B * C, T), cand_ent.reshape(B * C, T), p, c, windows).view(B, C, -1)
    hv = kcnn(clicked_title.reshape(B * H, T), clicked_ent.reshape(B * H, T), p, c, windows).view(B, H, -1)
    u = user_vector(hv, p)
    Fp = cv.shape[2]
    logits = score(cv.reshape(B * C, Fp), u.repeat_interleave(C, dim=0), p).view(B, C)
    return logits, cv, hv, u


def get_prediction(cand, clicked, p, windows=WINDOWS):
    """__init__.py:90-104: cand (n, F'), clicked (H, F') -> (n,), F' = len(windows) * F."""
    Fp = len(windows) * p["kcnn.additive_attention.linear.weight"].shape[1]
    if cand.shape[-1] != Fp or clicked.shape[-1] != Fp:
        raise ValueError(f"news vectors of width {cand.shape[-1]} / {clicked.shape[-1]} for {len(windows)} windows of {Fp // len(windows)}")
    u = user_vector(clicked.unsqueeze(0), p)
    return score(cand, u.expand(cand.shape[0], -1), p)
