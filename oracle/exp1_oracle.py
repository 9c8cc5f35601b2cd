"""CPU oracle for Exp1 (reference src/model/Exp1/**), built from the blocks of newsrec_oracle.py and held to the same
rules: TEST INFRASTRUCTURE ONLY, a plain torch-CPU restatement whose backward is autograd, pinned against golden vectors
of the live reference (oracle/make_golden_exp1.py -> tests/golden/exp1.npz).

Exp1 is NRMS with two more news views and a positional user input:
    news  title  -> NRMS news encoder (embedding, dropout, MHSA, dropout, additive pooling)      news_encoder.py:10-36
          category, subcategory -> relu(Linear(Embedding(id))), one shared category table      news_encoder.py:39-47, 70-79
          the stacked views -> additive attention (final_attention)                             news_encoder.py:80-110
    user  MHSA(hv + position_embedding) -> additive pooling                                    user_encoder.py:20-30

Storage contracts (the `contract` argument; DESIGN.md section 4):
    O.EXACT, O.WEIGHTS_BF16   one Contract everywhere (fp32 reference / the blueprint's tolerance definition);
    "fast"       every activation bf16 (O.BF16): title view, element views, the stacked views and hv + pos;
    "accurate"   title view as NRMS's accurate news encoder (O.BF16_FUSED); element views O.BF16 (fp32 output, bf16
                 pre-activation gradient); the stacked views as a hi/lo bf16 pair with a bf16 gradient, the final attention's
                 score GEMM on the hi plane and its pooled sum on both (O.BF16_FUSED); the user level fp32-accurate
                 (O.WEIGHTS_BF16) with pos added in fp32 and never rounded as an operand; dpos = sum of the input gradient.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

import newsrec_oracle as O

EXP1_VIEW_ORDER = ("title", "category", "subcategory")  # the reference's order follows a Python set; the fusion is
                                                       # permutation invariant up to fp summation order


def exp1_shapes(V, ncat, H, d=300, q=200, cat_dim=100):
    pre = "news_encoder.text_encoders.title"
    s = {f"{pre}.word_embedding.weight": (V, d)}
    for enc in (pre, "user_encoder"):
        for n in "QKV":
            s[f"{enc}.multihead_self_attention.W_{n}.weight"] = (d, d)
            s[f"{enc}.multihead_self_attention.W_{n}.bias"] = (d,)
    s.update(O._additive_shapes(f"{pre}.additive_attention", q, d))
    for name in ("category", "subcategory"):
        e = f"news_encoder.element_encoders.{name}"
        s[f"{e}.embedding.weight"] = (ncat, cat_dim)
        s[f"{e}.linear.weight"] = (d, cat_dim)
        s[f"{e}.linear.bias"] = (d,)
    s.update(O._additive_shapes("news_encoder.final_attention", q, d))
    s["user_encoder.position_embedding"] = (H, d)
    s.update(O._additive_shapes("user_encoder.additive_attention", q, d))
    return s


def exp1_state_dict(V, ncat, H, seed):
    """det_state_dict with the reference's U(-0.1, 0.1) init scale of the position embedding (user_encoder.py:14-16) and the
    shared category table under both element-encoder keys."""
    return O.tie_shared(O.det_state_dict(exp1_shapes(V, ncat, H), seed, {"user_encoder.position_embedding": 0.1}))


class _PoolHiGrad(torch.autograd.Function):
    """out = w . x over a hi/lo input x; the gradient of the pooling weights reads the hi plane, as the kernels' backward
    (nr_additive_attention_bwd on X_bf16) does."""

    @staticmethod
    def forward(ctx, w, x, x_hi):
        ctx.save_for_backward(w, x_hi)
        return torch.bmm(w.unsqueeze(1), x).squeeze(1)

    @staticmethod
    def backward(ctx, g):
        w, x_hi = ctx.saved_tensors
        return torch.bmm(x_hi, g.unsqueeze(-1)).squeeze(-1), w.unsqueeze(-1) * g.unsqueeze(1), None


def final_attention_hilo(x, p, prefix):
    """additive_attention (additive.py:27-53) on a hi/lo input: scores from the hi plane, pooled sum of both planes, backward
    on the hi plane with a bf16 pre-activation gradient."""
    c = O.BF16_FUSED
    xs = c.operand(x)
    pre = c.grad(F.linear(xs, c.operand(p[f"{prefix}.linear.weight"])) + p[f"{prefix}.linear.bias"])
    weights = F.softmax(torch.matmul(torch.tanh(pre), p[f"{prefix}.attention_query_vector"]), dim=1)
    return _PoolHiGrad.apply(weights, x, xs.detach())


def _contracts(contract):
    """-> (title, element views, stacked views (value -> value), final attention, user level)"""
    if contract == "accurate":
        return O.BF16_FUSED, O.BF16, O._RoundHiLo.apply, O.BF16_FUSED, O.WEIGHTS_BF16
    if contract == "fast":
        return O.BF16, O.BF16, O.BF16.act, O.BF16, O.BF16
    return contract, contract, contract.act, contract, contract


def exp1_news_encoder(news, p, heads=15, contract=O.EXACT, prefix="news_encoder", drop=None):
    """news_encoder.py:80-110 over {name: (n, ...)}; drop: nrms_news_encoder's train-mode masks for the title view."""
    c_title, c_elem, stack, c_final, _ = _contracts(contract)
    vecs = []
    for name in EXP1_VIEW_ORDER:
        if name not in news:
            continue
        if name == "title":
            vecs.append(O.nrms_news_encoder(news[name], p, heads, c_title, f"{prefix}.text_encoders.title", drop))
        else:
            vecs.append(O.naml_element_encoder(news[name], p, f"{prefix}.element_encoders.{name}", c_elem))
    if len(vecs) == 1:
        return vecs[0]
    if contract == "accurate":
        return final_attention_hilo(stack(torch.stack(vecs, dim=1)), p, f"{prefix}.final_attention")
    return O.additive_attention(stack(torch.stack(vecs, dim=1)), p, f"{prefix}.final_attention", c_final)


def exp1_user_encoder(hv, p, heads=15, contract=O.EXACT, prefix="user_encoder"):
    """user_encoder.py:20-30: the position embedding is broadcast over the batch (expand_as) and added before the MHSA."""
    c = _contracts(contract)[4]
    x = c.act(hv + p[f"{prefix}.position_embedding"])
    x = O.multihead_self_attention(x, p, f"{prefix}.multihead_self_attention", heads, c)
    return O.additive_attention(x, p, f"{prefix}.additive_attention", c)


def exp1_forward(cand, clicked, p, heads=15, contract=O.EXACT, drop=None):
    """__init__.py:15-45.  cand / clicked: {name: (B, C|H, ...)}.  drop=dict(p, seed): train mode with the kernels' masks (one
    title-encoder call over the browsed block, then the candidates, as the drop-in packs the batch)."""
    B, C = cand["title"].shape[:2]
    H = clicked["title"].shape[1]
    T = cand["title"].shape[2]
    flat = lambda dct, n: {k: v.reshape(B * n, *v.shape[2:]) for k, v in dct.items()}
    d_h = d_c = None
    if drop is not None:
        ld = (p["news_encoder.text_encoders.title.word_embedding.weight"].shape[1] + 8) // 8 * 8
        d_h, d_c = dict(drop, ld=ld, row0=0), dict(drop, ld=ld, row0=B * H * T)
    cv = exp1_news_encoder(flat(cand, C), p, heads, contract, drop=d_c).view(B, C, -1)
    hv = exp1_news_encoder(flat(clicked, H), p, heads, contract, drop=d_h).view(B, H, -1)
    return O.dot_product_click_predictor(cv, exp1_user_encoder(hv, p, heads, contract))


def ensemble_loss(logits_list):
    """train.py:192-200, 204-206: NLLLoss(log(mean_i softmax(logits_i))) with label 0."""
    mean = torch.stack([F.softmax(x, dim=1) for x in logits_list], dim=-1).mean(dim=-1)
    return F.nll_loss(torch.log(mean), torch.zeros(mean.shape[0], dtype=torch.long, device=mean.device))
