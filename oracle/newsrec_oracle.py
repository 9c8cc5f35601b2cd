"""CPU oracle for the NRMS / NAML / LSTUR / TANR forward+backward hot path.

TEST INFRASTRUCTURE ONLY.  Nothing under ``oracle/`` is imported by the product
package (``news-recommendation_b200/``); only ``tests/``, ``__graft_entry__.smoke()``
and ``bench.py``'s ``cpu_baseline`` / ``--impl reference`` legs may import it, and
there only as the checker / the CPU baseline, never as the thing shipped.

What it is: a plain torch-CPU functional restatement of the reference's algorithm
(the reference is pure Python/PyTorch, so a floating-point torch restatement is the
right oracle; see SURVEY.md section 8c).  Every function cites the reference
file:line it follows (paths relative to /root/reference).  Backward is torch
autograd over this restatement, which is exactly what the reference's
``loss.backward()`` (src/train.py:231) does.

Pinning: the reference holds NO golden vectors or tests for this path
(SURVEY.md section 4), so the oracle is pinned against outputs of the live
reference modules run in the build container: ``oracle/make_golden.py`` imports
``/root/reference/src`` and writes ``tests/golden/*.npz``;
``tests/test_oracle_golden.py`` checks this file against them (fp32, <=2e-6).

The bf16 contract: the CUDA path stores its large intermediates (gathered rows,
Q|K|V, attention context, and their gradients) in bf16 and feeds bf16 operands to
the tensor cores with fp32 accumulation.  ``Contract(bf16=True)`` inserts a
round-to-nearest-even bf16 rounding at exactly those points (forward values AND
the gradients flowing back through them), so that "kernel vs oracle" isolates
kernel bugs from the (documented) bf16 storage error.  ``Contract(bf16=False)`` is
the exact fp32/fp64 restatement of the reference.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import torch
import torch.nn.functional as F


# --------------------------------------------------------------------------- #
# bf16 storage contract
# --------------------------------------------------------------------------- #
def _round_bf16(x: torch.Tensor) -> torch.Tensor:
    return x.to(torch.bfloat16).to(x.dtype)


class _RoundBoth(torch.autograd.Function):
    """value -> bf16 on the way forward, gradient -> bf16 on the way back."""

    @staticmethod
    def forward(ctx, x):
        return _round_bf16(x)

    @staticmethod
    def backward(ctx, g):
        return _round_bf16(g)


class _RoundFwd(torch.autograd.Function):
    """value -> bf16 forward; gradient passes unrounded (fp32 accumulation)."""

    @staticmethod
    def forward(ctx, x):
        return _round_bf16(x)

    @staticmethod
    def backward(ctx, g):
        return g


class _RoundGrad(torch.autograd.Function):
    """identity forward; gradient -> bf16 on the way back."""

    @staticmethod
    def forward(ctx, x):
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        return _round_bf16(g)


class _RoundHiLo(torch.autograd.Function):
    """value -> bf16 hi + bf16 lo pair (about 16 mantissa bits) forward; gradient -> bf16 on the way back."""

    @staticmethod
    def forward(ctx, x):
        hi = _round_bf16(x)
        return hi + _round_bf16(x - hi)

    @staticmethod
    def backward(ctx, g):
        return _round_bf16(g)


@dataclass(frozen=True)
class Contract:
    bf16: bool = False
    hilo: bool = False     # precise storage: V and the context are hi/lo bf16 pairs
    acts: bool = True      # False: ONLY parameters / embeddings are rounded to bf16, every activation and gradient stays fp32
                           # (the tolerance definition of SURVEY.md 7.3-5: "the fp32 oracle on bf16-rounded weights/embeddings")

    def act(self, x):      # an activation the kernels store in bf16 (and whose grad they store in bf16)
        return _RoundBoth.apply(x) if (self.bf16 and self.acts) else x

    def act_hilo(self, x):  # an activation the fused kernels keep as a hi/lo bf16 pair (plain bf16 on the unfused path)
        if self.bf16 and self.hilo and self.acts:
            return _RoundHiLo.apply(x)
        return self.act(x)

    def operand(self, x):  # a parameter / input converted to a bf16 tensor-core operand; grad stays fp32
        return _RoundFwd.apply(x) if self.bf16 else x

    def grad(self, x):     # an fp32 value whose gradient the kernels store in bf16
        return _RoundGrad.apply(x) if (self.bf16 and self.acts) else x


EXACT = Contract(False)
BF16 = Contract(True)
BF16_FUSED = Contract(True, True)
WEIGHTS_BF16 = Contract(True, False, False)   # bf16 operands (weights, embedding table), fp32 everything else


# --------------------------------------------------------------------------- #
# dropout: NumPy restatement of the kernels' counter hash and mask (csrc/nr_common.cuh dropout_bits4
# and Dropout).  The reference draws its masks from torch's global RNG
# (news_encoder.py:38,43), which no kernel can reproduce; train-mode parity is therefore checked by
# giving the ORACLE the kernel's masks: element (row, col) of a matrix with pitch ld belongs to group
# (row*ld + col) >> 2 and is kept iff 16-bit lane (col & 3) of hash(seed, group) >= round(p * 65536).
# --------------------------------------------------------------------------- #
def dropout_bits4(seed: int, group):
    import numpy as np
    M32 = np.uint64(0xFFFFFFFF)
    group = np.asarray(group, dtype=np.uint64)
    s_lo, s_hi = np.uint64(seed & 0xFFFFFFFF), np.uint64((seed >> 32) & 0xFFFFFFFF)
    g_lo, g_hi = group & M32, group >> np.uint64(32)
    with np.errstate(over="ignore"):
        x = ((g_lo ^ s_lo) + g_hi * np.uint64(0x85EBCA6B) + s_hi * np.uint64(0x165667B1)) & M32
        x = (x * np.uint64(0x9E3779B1)) & M32
        x ^= x >> np.uint64(15)
        x = (x * np.uint64(0x85EBCA77)) & M32
        x ^= x >> np.uint64(13)
        y = (x * np.uint64(0xC2B2AE3D) + s_hi) & M32
        y ^= y >> np.uint64(16)
        y = (y * np.uint64(0x27D4EB2F)) & M32
        y ^= y >> np.uint64(15)
    return (y << np.uint64(32)) | x


def dropout_mask(seed: int, p: float, n_rows: int, n_cols: int, ld: int, row0: int = 0, col0: int = 0):
    """fp32 (n_rows, n_cols) multipliers (0 or 1/(1-p)) of rows [row0, row0+n_rows), columns [col0, col0+n_cols)."""
    import numpy as np
    if p <= 0.0:
        return torch.ones(n_rows, n_cols)
    assert ld % 4 == 0
    thresh = int(np.float32(p) * np.float32(65536.0) + np.float32(0.5))
    rows = (np.arange(n_rows, dtype=np.uint64) + np.uint64(row0))[:, None]
    cols = (np.arange(n_cols, dtype=np.uint64) + np.uint64(col0))[None, :]
    flat = rows * np.uint64(ld) + cols
    bits = dropout_bits4(seed, flat >> np.uint64(2))
    lane = (bits >> (np.uint64(16) * (flat & np.uint64(3)))) & np.uint64(0xFFFF)
    scale = np.float32(1.0) / (np.float32(1.0) - np.float32(p))
    return torch.from_numpy(np.where(lane >= thresh, scale, np.float32(0.0)).astype(np.float32))


# --------------------------------------------------------------------------- #
# shared modules  (reference: src/model/general/**)
# --------------------------------------------------------------------------- #
def scaled_dot_product_attention(Q, K, V, c: "Contract" = None):
    """src/model/general/attention/multihead_self.py:15-23.

    scores = exp(QK^T/sqrt(d_k)) WITHOUT max-subtraction; attn = scores/(sum+1e-8);
    no mask (no caller passes `length`, SURVEY.md 7.3-3).
    Contract: the attention probabilities enter the A.V product as bf16 tensor-core operands, and the
    gradient w.r.t. the scaled scores is rounded to bf16 (operand of the dQ / dK products); the softmax
    arithmetic itself is fp32.
    """
    d_k = Q.shape[-1]
    raw = torch.matmul(Q, K.transpose(-1, -2))
    if c is not None:
        raw = c.grad(raw)  # the kernels round dS/sqrt(d_k), i.e. the gradient w.r.t. the UNscaled product
    scores = torch.exp(raw / math.sqrt(d_k))
    attn = scores / (torch.sum(scores, dim=-1, keepdim=True) + 1e-8)
    if c is not None:
        if c.acts:  # P is an activation: it stays fp32 under the weights-only contract; the fused kernels keep it as a hi/lo pair
            attn = _RoundHiLo.apply(attn) if c.hilo else c.operand(attn)
    return torch.matmul(attn, V)


def multihead_self_attention(x, p, prefix, heads, c: Contract = EXACT, ctx_mask=None):
    """src/model/general/attention/multihead_self.py:46-76 (Q=K=V=x, length=None).

    x: (N, T, d).  W_Q/W_K/W_V are nn.Linear(d, d) WITH bias (:35-37); there is no
    output projection.  Contract: x is already a bf16 activation; the packed
    Q|K|V projection result is stored bf16; the per-head context is stored bf16.
    """
    N, T, d = x.shape
    d_k = d // heads

    def proj(name):
        w = c.operand(p[f"{prefix}.W_{name}.weight"])
        y = F.linear(x, w) + p[f"{prefix}.W_{name}.bias"]
        return c.act_hilo(y) if name == "V" else c.act(y)  # fused path: V enters P.V as a hi/lo pair

    def split(t):  # (N,T,d) -> (N,h,T,d_k)   (:53-58)
        return t.view(N, T, heads, d_k).transpose(1, 2)

    ctx = scaled_dot_product_attention(split(proj("Q")), split(proj("K")), split(proj("V")), c)
    ctx = ctx.transpose(1, 2).contiguous().view(N, T, d)  # (:74-76)
    if ctx_mask is not None:  # train mode: dropout on the context (NRMS/news_encoder.py:43) with an injected mask
        if not (c.bf16 and c.hilo):
            ctx = c.act(ctx)  # the unfused attention kernel rounds the context to bf16 BEFORE the 1/(1-p) scaling (and again after)
        ctx = ctx * ctx_mask
    return c.act_hilo(ctx)


def additive_attention(x, p, prefix, c: Contract = EXACT):
    """src/model/general/attention/additive.py:27-53.

    temp = tanh(linear(x)); w = softmax(temp @ q, dim=1); out = bmm(w, x).
    Contract: x is a bf16 activation; the linear runs on bf16 operands with fp32
    accumulation; tanh / score / softmax / weighted sum are fp32; the gradient
    w.r.t. the pre-activation is stored bf16.
    """
    w = c.operand(p[f"{prefix}.linear.weight"])
    xs = c.operand(x) if (c.bf16 and c.hilo and c.acts) else x  # hi/lo input: the score GEMM reads the hi plane, the pooled sum both
    pre = c.grad(F.linear(xs, w) + p[f"{prefix}.linear.bias"])
    temp = torch.tanh(pre)
    weights = F.softmax(torch.matmul(temp, p[f"{prefix}.attention_query_vector"]), dim=1)
    return torch.bmm(weights.unsqueeze(1), x).squeeze(1)


def dot_product_click_predictor(cand, user):
    """src/model/general/click_predictor/dot_product.py:8-19 (raw logits)."""
    return torch.bmm(cand, user.unsqueeze(-1)).squeeze(-1)


def embedding(ids, table, c: Contract = EXACT):
    """nn.Embedding lookup (e.g. src/model/NRMS/news_encoder.py:38).  Row 0's VALUE is
    used as-is; padding_idx=0 only suppresses its gradient (SURVEY.md 7.3-3e)."""
    return F.embedding(ids, c.operand(table), padding_idx=0)


def title_cnn(x, weight, bias, c: Contract = EXACT, y_mask=None):
    """Conv2d(1, F, (window, d), padding=((window-1)/2, 0)) over tokens + ReLU.
    src/model/NAML/news_encoder.py:15-17,27-32; LSTUR/news_encoder.py:24-28,60-66;
    TANR/news_encoder.py:21-25,43-48.  x: (N, T, d) -> (N, T, F).
    Contract: x is a bf16 activation, weight a bf16 operand; output stored bf16.
    y_mask (N, T, F): train mode, the dropout after the ReLU (e.g. NAML/news_encoder.py:33-34) with an injected mask --
    the kernel applies it in fp32 before the one bf16 store."""
    window = weight.shape[2]
    y = F.conv2d(x.unsqueeze(1), c.operand(weight), bias, padding=((window - 1) // 2, 0)).squeeze(3)
    y = F.relu(y).transpose(1, 2)
    if y_mask is not None:
        y = y * y_mask.to(y.dtype)
    return c.act_hilo(y)  # plain bf16 store; hi/lo pair under the accurate contract (LSTUR, config.precision)


def cnn_text_encoder(ids, table, conv_w, conv_b, p, att_prefix, c: Contract = EXACT, drop=None):
    """embedding -> dropout -> Conv2d + ReLU -> dropout -> additive pooling: the text encoder NAML, LSTUR and TANR share
    (NAML/news_encoder.py:21-37, LSTUR/news_encoder.py:56-72, TANR/news_encoder.py:40-52).
    drop=None: eval mode.  drop=dict(p, seed, n0): train mode with the kernels' masks -- the gathered rows live in the
    zero-padded layout (title n, token t -> row (n0+n)*(T+2) + 1 + t, pitch round_up(d+1, 8)) under hash(seed); the conv
    output in the compact layout (row (n0+n)*T + t, pitch round_up(F+1, 8)) under hash(seed ^ 0x5bd1e995); n0 = index of
    the first title of `ids` in the order the drop-in packs the batch (browsed block, then candidates)."""
    x = embedding(ids, table, c)
    y_mask = None
    if drop is not None and drop["p"] > 0:
        N, T, d = x.shape
        Fn = conv_w.shape[0]
        ru8 = lambda v: (v + 7) // 8 * 8
        n0 = drop.get("n0", 0)
        mx = dropout_mask(drop["seed"], drop["p"], N * (T + 2), d, ru8(d + 1), n0 * (T + 2)).view(N, T + 2, d)[:, 1:T + 1]
        y_mask = dropout_mask(drop["seed"] ^ 0x5bd1e995, drop["p"], N * T, Fn, ru8(Fn + 1), n0 * T).view(N, T, Fn)
        x = c.act(x * mx.to(x.dtype))
    y = title_cnn(x, conv_w, conv_b, c, y_mask)
    return additive_attention(y, p, att_prefix, c)


# --------------------------------------------------------------------------- #
# NRMS  (reference: src/model/NRMS/**)
# --------------------------------------------------------------------------- #
def nrms_news_encoder(title, p, heads, c: Contract = EXACT, prefix="news_encoder", drop=None):
    """src/model/NRMS/news_encoder.py:27-48.  drop=None: eval mode (dropout off, :38-45).
    drop=dict(p, seed, ld, row0): train mode with the kernels' masks -- embedding rows under hash(seed) (:38),
    context under hash(seed ^ 0x5bd1e995) (:43); rows are numbered row0.. in the order of `title`."""
    x = embedding(title, p[f"{prefix}.word_embedding.weight"], c)
    ctx_mask = None
    if drop is not None and drop["p"] > 0:
        N, T, d = x.shape
        mx = dropout_mask(drop["seed"], drop["p"], N * T, d, drop["ld"], drop.get("row0", 0)).view(N, T, d)
        ctx_mask = dropout_mask(drop["seed"] ^ 0x5bd1e995, drop["p"], N * T, d, drop["ld"], drop.get("row0", 0)).view(N, T, d)
        x = c.act(x * mx.to(x.dtype))  # the gathered rows are stored bf16 after the 1/(1-p) scaling
        ctx_mask = ctx_mask.to(x.dtype)
    x = multihead_self_attention(x, p, f"{prefix}.multihead_self_attention", heads, c, ctx_mask)
    return additive_attention(x, p, f"{prefix}.additive_attention", c)


def nrms_user_encoder(clicked_vec, p, heads, c: Contract = EXACT, prefix="user_encoder"):
    """src/model/NRMS/user_encoder.py:15-26."""
    x = c.act(clicked_vec)  # the kernel path re-stores the (B,H,d) news vectors as bf16 rows
    x = multihead_self_attention(x, p, f"{prefix}.multihead_self_attention", heads, c)
    return additive_attention(x, p, f"{prefix}.additive_attention", c)


def nrms_forward(cand_title, clicked_title, p, heads, c: Contract = EXACT, c_news: Contract = None, drop=None):
    """src/model/NRMS/__init__.py:19-48.  cand_title (B,C,T), clicked_title (B,H,T) int64.
    c_news: storage contract of the news encoder when it differs from the user encoder's (fused front end).
    drop: see nrms_news_encoder; rows are numbered as the drop-in packs them (browsed block, then candidates)."""
    B, C, T = cand_title.shape
    H = clicked_title.shape[1]
    cn = c if c_news is None else c_news
    d_clicked = None if drop is None else dict(drop, row0=0)
    d_cand = None if drop is None else dict(drop, row0=B * H * T)
    cand = nrms_news_encoder(cand_title.reshape(B * C, T), p, heads, cn, drop=d_cand).view(B, C, -1)
    clicked = nrms_news_encoder(clicked_title.reshape(B * H, T), p, heads, cn, drop=d_clicked).view(B, H, -1)
    user = nrms_user_encoder(clicked, p, heads, c)
    return dot_product_click_predictor(cand, user)


# --------------------------------------------------------------------------- #
# NAML  (reference: src/model/NAML/**)
# --------------------------------------------------------------------------- #
def naml_text_encoder(ids, p, prefix, c: Contract = EXACT, drop=None):
    """src/model/NAML/news_encoder.py:21-37 (drop: see cnn_text_encoder)."""
    return cnn_text_encoder(ids, p[f"{prefix}.word_embedding.weight"], p[f"{prefix}.CNN.weight"], p[f"{prefix}.CNN.bias"], p,
                            f"{prefix}.additive_attention", c, drop)


def naml_element_encoder(ids, p, prefix, c: Contract = EXACT):
    """src/model/NAML/news_encoder.py:46-47: relu(linear(embedding(id)))."""
    e = F.embedding(ids, c.operand(p[f"{prefix}.embedding.weight"]), padding_idx=0)
    w = c.operand(p[f"{prefix}.linear.weight"])
    return F.relu(c.grad(F.linear(e, w) + p[f"{prefix}.linear.bias"]))  # kernel stores d(pre-activation) in bf16


NAML_VIEW_ORDER = ("title", "abstract", "category", "subcategory")


def naml_news_encoder(news, p, c: Contract = EXACT, prefix="news_encoder", drop=None):
    """src/model/NAML/news_encoder.py:86-115.  The reference's view order follows a
    Python set (PYTHONHASHSEED dependent, SURVEY.md 7.3-9); the additive fusion is
    permutation invariant up to fp summation order, so a fixed order is used."""
    vecs = []
    for name in NAML_VIEW_ORDER:
        if name not in news:
            continue
        if name in ("title", "abstract"):
            d_view = None if drop is None else dict(p=drop["p"], seed=drop["seeds"][name], n0=drop.get("n0", 0))
            vecs.append(naml_text_encoder(news[name], p, f"{prefix}.text_encoders.{name}", c, d_view))
        else:
            vecs.append(naml_element_encoder(news[name], p, f"{prefix}.element_encoders.{name}", c))
    if len(vecs) == 1:
        return vecs[0]
    stacked = c.act(torch.stack(vecs, dim=1))
    return additive_attention(stacked, p, f"{prefix}.final_attention", c)


def naml_forward(cand, clicked, p, c: Contract = EXACT, drop=None):
    """src/model/NAML/__init__.py:19-54.  cand/clicked: dict name -> (B,C,..)/(B,H,..).
    drop=dict(p, seeds={"title": s1, "abstract": s2}): train mode with the kernels' masks (one seed per text encoder call)."""
    B, C = cand["title"].shape[:2]
    H = clicked["title"].shape[1]
    flat = lambda d, n: {k: v.reshape(B * n, *v.shape[2:]) for k, v in d.items()}
    d_h = None if drop is None else dict(drop, n0=0)
    d_c = None if drop is None else dict(drop, n0=B * H)
    cv = naml_news_encoder(flat(cand, C), p, c, drop=d_c).view(B, C, -1)
    hv = naml_news_encoder(flat(clicked, H), p, c, drop=d_h).view(B, H, -1)
    user = additive_attention(c.act(hv), p, "user_encoder.additive_attention", c)  # NAML/user_encoder.py:11-19
    return dot_product_click_predictor(cv, user)


# --------------------------------------------------------------------------- #
# TANR  (reference: src/model/TANR/**)
# --------------------------------------------------------------------------- #
def tanr_news_encoder(title, p, c: Contract = EXACT, prefix="news_encoder", drop=None):
    """src/model/TANR/news_encoder.py:30-54 (drop: see cnn_text_encoder)."""
    return cnn_text_encoder(title, p[f"{prefix}.word_embedding.weight"], p[f"{prefix}.title_CNN.weight"],
                            p[f"{prefix}.title_CNN.bias"], p, f"{prefix}.title_attention", c, drop)


def tanr_forward(cand, clicked, p, c: Contract = EXACT, drop=None):
    """src/model/TANR/__init__.py:24-69.  Returns (logits, topic_classification_loss).  drop=dict(p, seed): train mode."""
    B, C, T = cand["title"].shape
    H = clicked["title"].shape[1]
    d_h = None if drop is None else dict(drop, n0=0)
    d_c = None if drop is None else dict(drop, n0=B * H)
    cv = tanr_news_encoder(cand["title"].reshape(B * C, T), p, c, drop=d_c).view(B, C, -1)
    hv = tanr_news_encoder(clicked["title"].reshape(B * H, T), p, c, drop=d_h).view(B, H, -1)
    user = additive_attention(c.act(hv), p, "user_encoder.additive_attention", c)  # TANR/user_encoder.py:11-19
    logits = dot_product_click_predictor(cv, user)
    # :58-67  topic head over all B*(C+H) news vectors, class 0 has weight 0
    allv = torch.cat((cv, hv), dim=1).reshape(-1, cv.shape[-1])
    y_pred = c.grad(F.linear(c.operand(allv) if c.acts else allv, c.operand(p["topic_predictor.weight"])) + p["topic_predictor.bias"])
    y = torch.cat((cand["category"], clicked["category"]), dim=1).flatten()
    class_weight = torch.ones(y_pred.shape[1], dtype=y_pred.dtype)
    class_weight[0] = 0
    return logits, F.cross_entropy(y_pred, y, weight=class_weight)


# --------------------------------------------------------------------------- #
# LSTUR  (reference: src/model/LSTUR/**)
# --------------------------------------------------------------------------- #
def lstur_news_encoder(news, p, c: Contract = EXACT, prefix="news_encoder", drop=None):
    """src/model/LSTUR/news_encoder.py:32-76: [cat | subcat | title-CNN-pool] (drop: see cnn_text_encoder)."""
    catv = F.embedding(news["category"], p[f"{prefix}.category_embedding.weight"], padding_idx=0)
    subv = F.embedding(news["subcategory"], p[f"{prefix}.category_embedding.weight"], padding_idx=0)
    t = cnn_text_encoder(news["title"], p[f"{prefix}.word_embedding.weight"], p[f"{prefix}.title_CNN.weight"],
                         p[f"{prefix}.title_CNN.bias"], p, f"{prefix}.title_attention", c, drop)
    return torch.cat([catv, subv, t], dim=1)


def gru_last_hidden(x, lengths, h0, p, prefix, c: Contract = EXACT):
    """pack_padded_sequence(first len[b] steps, enforce_sorted=False) + nn.GRU, last hidden.
    src/model/LSTUR/user_encoder.py:27-45.  Gate order r,z,n (torch nn.GRU):
        r = sig(W_ir x + b_ir + W_hr h + b_hr); z likewise;
        n = tanh(W_in x + b_in + r*(W_hn h + b_hn)); h' = (1-z)*n + z*h.
    Row b stops updating after lengths[b] steps (packed-sequence semantics).
    Contract: x and h are bf16 operands of the two projections, gates fp32."""
    B, S, _ = x.shape
    w_ih = c.operand(p[f"{prefix}.weight_ih_l0"])
    w_hh = c.operand(p[f"{prefix}.weight_hh_l0"])
    b_ih, b_hh = p[f"{prefix}.bias_ih_l0"], p[f"{prefix}.bias_hh_l0"]
    Hd = w_hh.shape[1]
    # (B,S,3Hd); dX = dGI.W_ih stays fp32.  Under the accurate contract x enters as a hi/lo bf16 pair (~16 mantissa bits: not rounded here)
    gi_all = c.grad(F.linear(c.operand(x) if (c.acts and not c.hilo) else x, w_ih) + b_ih)
    h = h0
    for t in range(S):
        gh = c.grad(F.linear(c.operand(h) if (c.bf16 and c.acts) else h, w_hh) + b_hh)
        gi = gi_all[:, t]
        r = torch.sigmoid(gi[:, :Hd] + gh[:, :Hd])
        z = torch.sigmoid(gi[:, Hd:2 * Hd] + gh[:, Hd:2 * Hd])
        n = torch.tanh(gi[:, 2 * Hd:] + r * gh[:, 2 * Hd:])
        hn = (1 - z) * n + z * h
        active = (lengths > t).to(h.dtype).unsqueeze(1)
        h = active * hn + (1 - active) * h
    return h


def lstur_forward(user, lengths, cand, clicked, p, method="ini", c: Contract = EXACT, drop=None, user_keep=None):
    """src/model/LSTUR/__init__.py:44-87.  drop=None, user_keep=None: eval mode (== the get_user_vector path :89-108).
    drop=dict(p, seed): the title encoder's dropout with the kernels' masks; user_keep (B, 1): the multipliers of
    F.dropout2d on the (1, B, dim) user embedding (:74-77) == whole user vectors dropped with masking_probability and the
    rest scaled by 1/(1-p).  lengths==0 is clamped to 1 (user_encoder.py:27)."""
    B, C = cand["title"].shape[:2]
    H = clicked["title"].shape[1]
    flat = lambda d, n: {k: v.reshape(B * n, *v.shape[2:]) for k, v in d.items()}
    d_h = None if drop is None else dict(drop, n0=0)
    d_c = None if drop is None else dict(drop, n0=B * H)
    cv = lstur_news_encoder(flat(cand, C), p, c, drop=d_c).view(B, C, -1)
    hv = lstur_news_encoder(flat(clicked, H), p, c, drop=d_h).view(B, H, -1)
    uemb = F.embedding(user, p["user_embedding.weight"], padding_idx=0)
    if user_keep is not None:
        uemb = uemb * user_keep.to(uemb.dtype)
    lengths = lengths.clamp(min=1)
    if method == "ini":
        uv = gru_last_hidden(hv, lengths, uemb, p, "user_encoder.gru", c)
    else:
        h0 = torch.zeros(B, p["user_encoder.gru.weight_hh_l0"].shape[1], dtype=hv.dtype)
        uv = torch.cat((gru_last_hidden(hv, lengths, h0, p, "user_encoder.gru", c), uemb), dim=1)
    return dot_product_click_predictor(cv, uv)


# --------------------------------------------------------------------------- #
# loss  (reference: src/train.py:126,205-206 -- label is always index 0)
# --------------------------------------------------------------------------- #
def click_loss(logits):
    return F.cross_entropy(logits, torch.zeros(logits.shape[0], dtype=torch.long))


# --------------------------------------------------------------------------- #
# deterministic synthetic parameters / inputs (no dependence on torch/numpy RNG
# stream stability: splitmix64 hashing of the element index)
# --------------------------------------------------------------------------- #
def _splitmix64(x):
    import numpy as np
    x = (x + np.uint64(0x9E3779B97F4A7C15)) & np.uint64(0xFFFFFFFFFFFFFFFF)
    z = x
    z = ((z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)) & np.uint64(0xFFFFFFFFFFFFFFFF)
    z = ((z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)) & np.uint64(0xFFFFFFFFFFFFFFFF)
    return z ^ (z >> np.uint64(31))


def det_uniform(shape, seed, lo=-1.0, hi=1.0, dtype=torch.float32):
    """Deterministic U[lo,hi) tensor: value(i) = f(splitmix64(seed*2^32 + i)); stable forever."""
    import numpy as np
    n = int(np.prod(shape)) if len(shape) else 1
    with np.errstate(over="ignore"):
        idx = np.arange(n, dtype=np.uint64) + (np.uint64(seed) << np.uint64(32))
        bits = _splitmix64(idx)
    u = (bits >> np.uint64(11)).astype(np.float64) * (1.0 / (1 << 53))
    return torch.from_numpy((lo + (hi - lo) * u).reshape(shape)).to(dtype)


def det_randint(shape, seed, lo, hi):
    """Deterministic integers in [lo, hi)."""
    u = det_uniform(shape, seed, 0.0, 1.0, torch.float64)
    return (lo + (u * (hi - lo)).floor()).clamp(max=hi - 1).to(torch.int64)


def _str_seed(name: str) -> int:
    h = 1469598103
    for ch in name.encode():
        h = ((h ^ ch) * 16777619) & 0x7FFFFFFF
    return h


def det_state_dict(shapes: dict, seed: int, scale_overrides: dict | None = None):
    """A deterministic fp32 state_dict for the given {key: shape}.  Magnitudes follow the
    reference initialisers' scale (xavier-ish for matrices, small biases, N(0,1)-ish
    embeddings) so that activations are O(1) and exp() is well inside fp32 range."""
    out = {}
    for k, shp in shapes.items():
        s = (_str_seed(k) ^ (seed * 7919)) & 0x7FFFFFFF
        if scale_overrides and k in scale_overrides:
            a = scale_overrides[k]
        elif k.endswith("embedding.weight") or k.endswith("word_embedding.weight"):
            a = 1.0
        elif k.endswith("attention_query_vector"):
            a = 0.1
        elif "bias" in k:
            a = 0.05
        else:
            fan = 1
            for d in shp[1:]:
                fan *= d
            a = math.sqrt(6.0 / (fan + shp[0]))
        out[k] = det_uniform(tuple(shp), s, -a, a)
    return out


def nrms_shapes(V, d=300, q=200):
    s = {"news_encoder.word_embedding.weight": (V, d)}
    for enc in ("news_encoder", "user_encoder"):
        for n in "QKV":
            s[f"{enc}.multihead_self_attention.W_{n}.weight"] = (d, d)
            s[f"{enc}.multihead_self_attention.W_{n}.bias"] = (d,)
        s[f"{enc}.additive_attention.attention_query_vector"] = (q,)
        s[f"{enc}.additive_attention.linear.weight"] = (q, d)
        s[f"{enc}.additive_attention.linear.bias"] = (q,)
    return s


def _additive_shapes(prefix, q, dim):
    return {f"{prefix}.attention_query_vector": (q,), f"{prefix}.linear.weight": (q, dim),
            f"{prefix}.linear.bias": (q,)}


def naml_shapes(V, ncat, d=300, q=200, Fn=300, cat_dim=100, window=3):
    s = {}
    for name in ("title", "abstract"):
        pre = f"news_encoder.text_encoders.{name}"
        s[f"{pre}.word_embedding.weight"] = (V, d)
        s[f"{pre}.CNN.weight"] = (Fn, 1, window, d)
        s[f"{pre}.CNN.bias"] = (Fn,)
        s.update(_additive_shapes(f"{pre}.additive_attention", q, Fn))
    for name in ("category", "subcategory"):
        pre = f"news_encoder.element_encoders.{name}"
        s[f"{pre}.embedding.weight"] = (ncat, cat_dim)
        s[f"{pre}.linear.weight"] = (Fn, cat_dim)
        s[f"{pre}.linear.bias"] = (Fn,)
    s.update(_additive_shapes("news_encoder.final_attention", q, Fn))
    s.update(_additive_shapes("user_encoder.additive_attention", q, Fn))
    return s


def tanr_shapes(V, ncat, d=300, q=200, Fn=300, window=3):
    s = {"news_encoder.word_embedding.weight": (V, d),
         "news_encoder.title_CNN.weight": (Fn, 1, window, d), "news_encoder.title_CNN.bias": (Fn,)}
    s.update(_additive_shapes("news_encoder.title_attention", q, Fn))
    s.update(_additive_shapes("user_encoder.additive_attention", q, Fn))
    s["topic_predictor.weight"] = (ncat, Fn)
    s["topic_predictor.bias"] = (ncat,)
    return s


def lstur_shapes(V, ncat, nusers, d=300, q=200, Fn=300, window=3, method="ini"):
    D = 3 * Fn
    Hd = D if method == "ini" else int(Fn * 1.5)
    s = {"news_encoder.word_embedding.weight": (V, d),
         "news_encoder.category_embedding.weight": (ncat, Fn),
         "news_encoder.title_CNN.weight": (Fn, 1, window, d), "news_encoder.title_CNN.bias": (Fn,)}
    s.update(_additive_shapes("news_encoder.title_attention", q, Fn))
    s.update({"user_encoder.gru.weight_ih_l0": (3 * Hd, D), "user_encoder.gru.weight_hh_l0": (3 * Hd, Hd),
              "user_encoder.gru.bias_ih_l0": (3 * Hd,), "user_encoder.gru.bias_hh_l0": (3 * Hd,),
              "user_embedding.weight": (nusers, Hd)})
    return s


def tie_shared(p: dict):
    """The reference shares ONE nn.Embedding object between NAML's text encoders and between
    its element encoders (src/model/NAML/news_encoder.py:55-61,71-80): same storage, two keys."""
    a, b = "news_encoder.text_encoders.title.word_embedding.weight", "news_encoder.text_encoders.abstract.word_embedding.weight"
    if a in p and b in p:
        p[b] = p[a]
    a, b = "news_encoder.element_encoders.category.embedding.weight", "news_encoder.element_encoders.subcategory.embedding.weight"
    if a in p and b in p:
        p[b] = p[a]
    return p


def synth_titles(n, T, V, seed, min_len=5):
    """MIND-like token ids: length U{min_len..T}, right-padded with 0 (SURVEY.md 8d)."""
    ids = det_randint((n, T), seed, 1, V)
    lens = det_randint((n,), seed + 1, min_len, T + 1)
    mask = torch.arange(T).unsqueeze(0) < lens.unsqueeze(1)
    return ids * mask


def synth_batch(B, C, H, T, V, seed, with_hist_pad=True):
    """(cand (B,C,T), clicked (B,H,T), hist_len (B,)); history LEFT-padded with all-zero news
    (src/dataset.py:82-83)."""
    cand = synth_titles(B * C, T, V, seed).view(B, C, T)
    clicked = synth_titles(B * H, T, V, seed + 10).view(B, H, T)
    hist_len = det_randint((B,), seed + 20, 1, H + 1) if with_hist_pad else torch.full((B,), H)
    keep = torch.arange(H).unsqueeze(0) >= (H - hist_len).unsqueeze(1)
    clicked = clicked * keep.unsqueeze(-1)
    return cand, clicked, hist_len


# --------------------------------------------------------------------------- #
# CPU baseline: the reference's NRMS training step, restated with the reference's OWN call structure
# (one news_encoder call per slot, dropout active in train mode, dense Embedding gradient), so that
# timing it is timing what the reference does on the host cores.  Used by bench.py (cpu_baseline /
# --impl reference) only.
# --------------------------------------------------------------------------- #
class ReferenceStructuredNRMS(torch.nn.Module):
    """src/model/NRMS/__init__.py:7-48 + news_encoder.py:27-48 + user_encoder.py:15-26, slot by slot."""

    def __init__(self, V, d=300, heads=15, q=200, p_drop=0.2, seed=0):
        super().__init__()
        self.heads, self.p_drop = heads, p_drop
        sd = det_state_dict(nrms_shapes(V, d, q), seed)
        self.params = torch.nn.ParameterDict({k.replace(".", "/"): torch.nn.Parameter(v) for k, v in sd.items()})

    def _p(self):
        return {k.replace("/", "."): v for k, v in self.params.items()}

    def news_encoder(self, title, p):
        # news_encoder.py:38-47 (dropout after the embedding and after the self-attention)
        x = F.dropout(embedding(title, p["news_encoder.word_embedding.weight"]), p=self.p_drop, training=self.training)
        x = multihead_self_attention(x, p, "news_encoder.multihead_self_attention", self.heads)
        x = F.dropout(x, p=self.p_drop, training=self.training)
        return additive_attention(x, p, "news_encoder.additive_attention")

    def forward(self, candidate_news, clicked_news):
        p = self._p()
        cand = torch.stack([self.news_encoder(x["title"], p) for x in candidate_news], dim=1)   # __init__.py:38-39
        clicked = torch.stack([self.news_encoder(x["title"], p) for x in clicked_news], dim=1)  # __init__.py:41-42
        user = nrms_user_encoder(clicked, p, self.heads)
        return dot_product_click_predictor(cand, user)


def reference_cpu_step(model, candidate_news, clicked_news):
    """zero_grad -> forward -> CrossEntropy(label 0) -> backward  (src/train.py:202-231, optimizer excluded:
    the metric is forward+backward)."""
    for prm in model.parameters():
        prm.grad = None
    loss = click_loss(model(candidate_news, clicked_news))
    loss.backward()
    return float(loss.detach())
