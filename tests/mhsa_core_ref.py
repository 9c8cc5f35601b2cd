"""fp64 references and per-element bounds of the self-attention core (nr_mhsa_core_fwd / _bwd, csrc/attn.cu and
csrc/attn_title.cu), as plain functions of tensors on any device.  tests/test_mhsa_core_host.py checks them against
torch.autograd through the oracle on the CPU; tests/test_gpu_mhsa_core.py holds the kernels to them (the bounds are derived
in its module docstring).

Layout: Q, K, V, dC are fp64 (n, T, d) tensors holding the bf16 values the kernels read, d = heads * d_k; head h owns columns
[h d_k, (h + 1) d_k)."""
from __future__ import annotations

import math

import torch

U32 = 2.0 ** -23      # one fp32 ulp, relative: the allowance of one fp32 accumulation step (tensor-core sums may truncate)
APPROX = 2.0 ** -20   # ex2.approx, the reciprocal and the few fp32 operations of the softmax normalisation, relative
TINY = 2.0 ** -100    # absolute: probabilities below the fp32 normal range flush to zero


def bf16(t):
    return t.to(torch.bfloat16).to(t.dtype)


def ulp(v):
    """One bf16 ulp at |v| (fp64 tensor); 0 where v == 0."""
    _, e = torch.frexp(v.abs())
    return torch.where(v == 0, torch.zeros_like(v), torch.ldexp(torch.ones_like(v), e - 8))


def split(t, heads):
    n, T, d = t.shape
    return t.reshape(n, T, heads, d // heads).transpose(1, 2)


def merge(t):
    n, h, T, dk = t.shape
    return t.transpose(1, 2).reshape(n, T, h * dk)


def scores(Q, K, heads):
    """S = Q_h K_h^T / sqrt(d_k): (n, heads, T, T)."""
    dk = Q.shape[2] // heads
    return split(Q, heads) @ split(K, heads).transpose(-1, -2) / math.sqrt(dk)


def probs(S, keys=None):
    """A = exp(S) / (sum_j exp(S) + 1e-8) (multihead_self.py:15-23) in its max-subtracted form; keys: use only the first
    `keys` key rows (a reference that leaves the last ones out)."""
    if keys is not None:
        S = S[..., :keys]
    m = S.amax(-1, keepdim=True)
    e = torch.exp(S - m)
    return e / (e.sum(-1, keepdim=True) + 1e-8 * torch.exp(-m))


def forward(Q, K, V, heads, keys=None):
    """The exact context A V (n, T, d) and A (n, heads, T, T)."""
    A = probs(scores(Q, K, heads), keys)
    Vh = split(V, heads)[..., :A.shape[-1], :]
    return merge(A @ Vh), A


def backward(Q, K, V, dC, heads, contract=False):
    """dQ, dK, dV (n, T, d) of the context A V with upstream gradient dC; dS is the gradient w.r.t. the UNscaled product Q K^T
    (what the kernels round, oracle.scaled_dot_product_attention).  contract=True: A enters dV and dS enters dQ, dK as bf16
    operands, as the kernels feed the tensor cores."""
    r = bf16 if contract else (lambda t: t)
    dk = Q.shape[2] // heads
    A = probs(scores(Q, K, heads))
    G = split(dC, heads)
    dA = G @ split(V, heads).transpose(-1, -2)
    dS = A * (dA - (A * dA).sum(-1, keepdim=True)) / math.sqrt(dk)
    return dict(dQ=merge(r(dS) @ split(K, heads)), dK=merge(r(dS).transpose(-1, -2) @ split(Q, heads)),
                dV=merge(r(A).transpose(-1, -2) @ G), A=A, dS=dS, dA=dA)


def prob_error(Q, K, heads):
    """Relative error bound eps (n, heads, T, T) of the kernels' fp32 probabilities (plus TINY absolute).  The scores carry the
    fp32 accumulation of d_k exact bf16 products (d_k U32 sum |q||k| / sqrt(d_k)) and the roundings of the scale and of the
    max-subtracted exponent argument (2^-21 of |S| and of |S - max S|); an error dS_j in score j moves A_ij by dS_j relatively
    and the normalisation by at most the row's largest dS; exp2, the row sum of T terms and the reciprocal add APPROX + T U32."""
    dk = Q.shape[2] // heads
    T = Q.shape[1]
    S = scores(Q, K, heads)
    absraw = split(Q.abs(), heads) @ split(K.abs(), heads).transpose(-1, -2)
    dS = dk * U32 * absraw / math.sqrt(dk) + 2.0 ** -21 * (S.abs() + (S.amax(-1, keepdim=True) - S))
    return dS + dS.amax(-1, keepdim=True) + APPROX + T * U32


def flip(x, dx):
    """The largest change of bf16(y) over |y - x| <= dx: 0 where no bf16 rounding boundary lies within dx of x."""
    r = bf16(x)
    return torch.maximum((bf16(x + dx) - r).abs(), (r - bf16(x - dx)).abs())


def context_bound(Q, K, V, heads, cm):
    """Per element of the context: A V (exact), the bound and its parts.  cm (n, T, d) are the dropout multipliers.
    bound = one bf16 ulp (two where the mask rescales: rounded before and after the 1/(1 - p) scaling)
            + sum_j (2^-8 + eps_ij) A_ij |V_j| m  (A enters A V as bf16; its fp32 error and the fp32 sum)  + TINY sum |V| m."""
    ctx, A = forward(Q, K, V, heads)
    eps = prob_error(Q, K, heads)
    Vh = split(V.abs(), heads)
    spread = merge(((2.0 ** -8 + eps) * A + TINY) @ Vh) * cm
    ref = ctx * cm
    return ref, spread


def judge_context(got, ref, spread, cm):
    """Worst |got - ref| / (ulps + spread) over the elements; NaN counts as +inf."""
    ulps = ulp(torch.maximum(got.abs(), ref.abs())) * torch.where(cm > 1, 2.0, 1.0)
    r = (got - ref).abs() / (ulps + spread)
    r = torch.where((got - ref) == 0, torch.zeros_like(r), r)
    return torch.nan_to_num(r, nan=float("inf"))


def grad_bounds(Q, K, V, dC, heads):
    """Contract references of dQ, dK, dV (bf16 dS / bf16 A operands) and their per-element spreads (without the half ulp of the
    output, which depends on the stored value):
      dV_j = sum_i bf16(A_ij) dC_i: the kernel's fp32 A is within eps A + TINY of A, so its bf16 rounding differs from bf16(A)
             by at most flip(A, eps A + TINY); plus T U32 sum_i |bf16(A_ij)| |dC_i| for the fp32 sum.
      dQ_i = sum_j bf16(dS_ij) K_j, dK_j = sum_i bf16(dS_ij) Q_i: the kernel's fp32 dS = A (dA - sum A dA) / sqrt(d_k) is within
             delta of the exact one, delta from eps of A, the fp32 sums of dA (d_k U32 sum |dC||V|) and of sum A dA, and 2^-21
             |dS| for the scaling; its bf16 rounding differs from bf16(dS) by at most flip(dS, delta); plus T U32 for the sum."""
    dk = Q.shape[2] // heads
    T = Q.shape[1]
    b = backward(Q, K, V, dC, heads, contract=True)
    A, dS, dA = b["A"], b["dS"], b["dA"]
    eps = prob_error(Q, K, heads)
    G = split(dC, heads)
    dA_err = dk * U32 * (G.abs() @ split(V.abs(), heads).transpose(-1, -2))
    dam = dA - (A * dA).sum(-1, keepdim=True)
    del_err = ((eps * A + TINY) * dA.abs() + A * dA_err).sum(-1, keepdim=True) + T * U32 * (A * dA.abs()).sum(-1, keepdim=True)
    delta = ((eps * A + TINY) * dam.abs() + (A + TINY) * (dA_err + del_err)) / math.sqrt(dk) + 2.0 ** -21 * dS.abs()
    fA = flip(A, eps * A + TINY)
    fS = flip(dS, delta)
    rA, rS = bf16(A), bf16(dS).abs()
    Kh, Qh = split(K.abs(), heads), split(Q.abs(), heads)
    spread = dict(dV=merge((fA + T * U32 * rA).transpose(-1, -2) @ G.abs()),
                  dQ=merge((fS + T * U32 * rS) @ Kh),
                  dK=merge((fS + T * U32 * rS).transpose(-1, -2) @ Qh))
    return dict(dQ=b["dQ"], dK=b["dK"], dV=b["dV"]), spread


def judge_grad(got, ref, spread):
    """Worst |got - ref| / (half an ulp + spread); NaN counts as +inf."""
    half = 0.5 * ulp(torch.maximum(got.abs(), ref.abs()))
    r = (got - ref).abs() / (half + spread)
    r = torch.where((got - ref) == 0, torch.zeros_like(r), r)
    return torch.nan_to_num(r, nan=float("inf"))


def neighbour_head(t, heads):
    """The tensor with head h's columns replaced by head (h + 1) mod heads's."""
    return merge(torch.roll(split(t, heads), -1, dims=1))
