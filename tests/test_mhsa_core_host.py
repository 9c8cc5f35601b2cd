"""Host-side checks of the self-attention core's references and bounds (no device needed).

* The fp64 references tests/test_gpu_mhsa_core.py holds the kernels to (tests/mhsa_core_ref.py: the stable-form forward and
  the dQ / dK / dV chain, exact and under the bf16 contract) against torch.autograd through oracle.scaled_dot_product_attention
  in fp64, in the unit-scale, saturated and strongly negative score regimes.
* The checker itself: an fp32 restatement of the kernels' arithmetic (fp32 scores of bf16 operands, the max-subtracted exp2
  softmax with the 1e-8 exp2(-max) term, bf16 probabilities and score gradients as MMA operands, bf16 outputs) passes every
  bound; the same arithmetic with one planted fault -- no 1e-8 term, one wrong row of one head, unrounded probabilities in
  dV -- fails its bound, and the discrimination references miss theirs by >= 8x."""
import math

import pytest
import torch

import gpu_checks as G
import mhsa_core_ref as R
import newsrec_oracle as O


def _inputs(n, T, heads, dk, regime, seed=3):
    return G.mhsa_core_inputs(n, T, heads, dk, regime, seed, device="cpu")


@pytest.mark.parametrize("regime", ["unit", "saturated", "negative"])
@pytest.mark.parametrize("T,heads,dk", [(7, 3, 5), (20, 2, 20), (1, 2, 4)])
def test_references_match_autograd_through_the_oracle(regime, T, heads, dk):
    Q, K, V, dC = _inputs(3, T, heads, dk, regime)
    rel = lambda a, b: float((a - b).norm() / max(float(b.norm()), 1e-300))
    for contract in (False, True):
        q, k, v = (R.split(t, heads).clone().requires_grad_(True) for t in (Q, K, V))
        out = O.scaled_dot_product_attention(q, k, v, O.BF16 if contract else None)
        out.backward(R.split(dC, heads))
        b = R.backward(Q, K, V, dC, heads, contract=contract)
        tol = 1e-6 if contract else 1e-10
        for key, t in (("dQ", q), ("dK", k), ("dV", v)):
            want = R.merge(t.grad)
            if T == 1 and key != "dV":  # dS = A (1 - A) dA / sqrt(d_k) ~ 1e-8 dA: compared on the scale of dA
                assert float((b[key] - want).abs().max()) <= 1e-14 * float(dC.abs().max() * V.abs().max() * Q.abs().max()), key
                continue
            assert rel(b[key], want) < tol, (key, contract, rel(b[key], want))
        if not contract:
            assert rel(R.forward(Q, K, V, heads)[0], R.merge(out.detach())) < 1e-10
    if regime == "negative":  # the +1e-8 dominates: the context is orders of magnitude below sum A |V| of a normalised softmax
        ctx, A = R.forward(Q, K, V, heads)
        assert float(A.sum(-1).max()) < 0.1


# ------------------------------------------------------------------------------------------------
def _emulate(Q, K, V, dC, heads, cm, fault=None):
    """The kernels' arithmetic in fp32 on the CPU (csrc/attn.cu softmax_rows and the two phases of the backward)."""
    bf = lambda t: t.to(torch.bfloat16).float()
    dk = Q.shape[2] // heads
    q, k, v, g = (R.split(t.float(), heads) for t in (Q, K, V, dC))
    sc = torch.tensor(1.4426950408889634 / math.sqrt(dk), dtype=torch.float32)
    rs = torch.tensor(1.0 / math.sqrt(dk), dtype=torch.float32)
    s = q @ k.transpose(-1, -2)
    m = s.amax(-1, keepdim=True) * sc
    e = torch.exp2(s * sc - m)
    corr = 0.0 if fault == "no_1e-8" else torch.tensor(1e-8, dtype=torch.float32) * torch.exp2(-m)
    P = e * (1.0 / (e.sum(-1, keepdim=True) + corr))
    ctx = R.merge(bf(bf(P) @ v)).double()
    if fault == "one_row":
        ctx[0, 1, dk:2 * dk] = ctx[0, 2, dk:2 * dk]
    ctx = torch.where(cm > 1, bf((ctx * cm).float()).double(), ctx * cm)
    dA = g @ v.transpose(-1, -2)
    dS = P * (dA - (P * dA).sum(-1, keepdim=True)) * rs
    Pv = P if fault == "unrounded_A" else bf(P)
    grads = dict(dQ=bf(bf(dS) @ k), dK=bf(bf(dS).transpose(-1, -2) @ q), dV=bf(Pv.transpose(-1, -2) @ g))
    return ctx, {key: R.merge(t).double() for key, t in grads.items()}


def _judge(Q, K, V, dC, heads, cm, ctx, grads):
    ref_c, spread_c = R.context_bound(Q, K, V, heads, cm)
    refs, spread = R.grad_bounds(Q, K, V, dC, heads)
    out = {"ctx": float(R.judge_context(ctx, ref_c, spread_c, cm).max())}
    for key in ("dQ", "dK", "dV"):
        out[key] = float(R.judge_grad(grads[key], refs[key], spread[key]).max())
    return out, ref_c, spread_c, spread


def _mask(n, T, d, seed=9, p=0.2):
    keep = O.det_uniform((n, T, d), seed, 0.0, 1.0) >= p
    return keep.double() / (1.0 - p)


@pytest.mark.parametrize("regime", ["unit", "saturated", "negative"])
@pytest.mark.parametrize("T,heads,dk", [(17, 3, 16), (20, 4, 20), (50, 2, 9), (64, 2, 32)])
def test_kernel_arithmetic_passes_every_bound(regime, T, heads, dk):
    Q, K, V, dC = _inputs(5, T, heads, dk, regime)
    cm = _mask(5, T, heads * dk)
    ctx, grads = _emulate(Q, K, V, dC, heads, cm)
    r, ref_c, spread_c, spread = _judge(Q, K, V, dC, heads, cm, ctx, grads)
    assert all(v <= 1.0 for v in r.values()), r
    # the discrimination references of the GPU test miss by far
    worst = lambda ref: float(R.judge_context(ctx, ref, spread_c, cm).max())
    assert worst(R.neighbour_head(ref_c, heads)) >= 8
    assert worst(R.forward(Q, K, V, heads, keys=T - 1)[0] * cm) >= 8
    assert worst(R.forward(Q, K, V, heads)[0] * _mask(5, T, heads * dk, seed=10)) >= 8
    if regime != "saturated":  # nearly one-hot rows: A rounds to 1 or is far below the output's ulp
        assert float(R.judge_grad(grads["dV"], R.backward(Q, K, V, dC, heads)["dV"], spread["dV"]).max()) >= 8


def test_flush_regime_gives_exact_zeros():
    """Every score below -95: exp2(-max) overflows to inf in fp32, the normaliser to 0, and so every output."""
    Q, K, V, dC = _inputs(3, 20, 2, 16, "flush")
    assert float(R.scores(Q, K, 2).max()) < -95
    ctx, grads = _emulate(Q, K, V, dC, 2, torch.ones(3, 20, 32, dtype=torch.float64))
    assert bool((ctx == 0).all()) and all(bool((g == 0).all()) for g in grads.values())


@pytest.mark.parametrize("fault,regime,stage", [("no_1e-8", "negative", "ctx"), ("one_row", "unit", "ctx"),
                                                ("unrounded_A", "unit", "dV")])
def test_planted_faults_fail_their_bound(fault, regime, stage):
    Q, K, V, dC = _inputs(5, 20, 3, 16, regime)
    cm = torch.ones(5, 20, 48, dtype=torch.float64)
    ctx, grads = _emulate(Q, K, V, dC, 3, cm, fault=fault)
    r = _judge(Q, K, V, dC, 3, cm, ctx, grads)[0]
    assert r[stage] > 1.0, r
