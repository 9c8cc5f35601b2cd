"""The additive-attention backward (nr_additive_attention_bwd: score gradient, the dPre GEMM and the input-gradient GEMM)
against an fp64 evaluation of the same bf16 operands, row by row.

The bf16 contract is applied at the points where the kernels round: the rows X and the weight Wa are bf16, dPre is rounded to
bf16 before it enters the input-gradient and weight-gradient products, and dX is stored as bf16.  The softmax weights w are
the ones the forward kernel saved, so the reference differs from the kernels only by fp32 accumulation order, the tanh
approximation and the rounding of dPre that follows from them (a dPre element may land one bf16 step away).

Shapes: the NRMS news level (seg 20, D 300, q 200), the user level (seg 50), Exp1's seg 3, and edges of the two epilogues:
rows not a multiple of the 64-row tile, a single tile, q below one 32-column chunk and q not a multiple of 16 (dPre leaves by
plain stores / a chunk cut by the query width), D = 64 and D = 320 (one weight slice, whole chunks), D = 296 (a chunk cut
by the slice end) and D = 400 (slices of 208 / 192 columns)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _bf16(t):
    return t.to(torch.bfloat16).to(torch.float32)


def _run(N, S, D, q, seed):
    from newsrec_b200.ops import AdditiveAttentionFn, OperandCache
    g = torch.Generator().manual_seed(seed)
    x = _bf16(torch.rand((N, S, D), generator=g) * 2 - 1)
    wa = torch.rand((q, D), generator=g) * 0.2 - 0.1
    ba = torch.rand((q,), generator=g) * 0.1 - 0.05
    qv = torch.rand((q,), generator=g) * 0.2 - 0.1
    dout = torch.rand((N, D), generator=g) * 2 - 1
    xd = x.to(DEV).requires_grad_(True)
    pd = [t.to(DEV).requires_grad_(True) for t in (wa, ba, qv)]
    out = AdditiveAttentionFn.apply(xd, pd[0], pd[1], pd[2], OperandCache(), "t", "fast")
    out.backward(dout.to(DEV))
    torch.cuda.synchronize()
    # the forward's own softmax weights (fp32) enter the reference: the backward is what is checked
    xf = x.double()
    waf = _bf16(wa).double()
    pre = torch.einsum("nsd,cd->nsc", xf, waf) + ba.double()
    t = torch.tanh(pre)
    w = torch.softmax(t @ qv.double(), dim=1)
    dw = torch.einsum("nsd,nd->ns", xf, dout.double())
    ds = w * (dw - (w * dw).sum(dim=1, keepdim=True))
    dpre = _bf16((ds[..., None] * qv.double() * (1 - t * t)).float()).double()
    dx = torch.einsum("nsc,cd->nsd", dpre, waf) + w[..., None] * dout.double()[:, None, :]
    dwa = torch.einsum("nsc,nsd->cd", dpre, xf)
    dba = dpre.sum(dim=(0, 1))
    dqv = torch.einsum("ns,nsc->c", ds, t)
    return {"dx": (xd.grad.double().cpu().reshape(N * S, D), dx.reshape(N * S, D)), "dWa": (pd[0].grad.double().cpu(), dwa),
            "dba": (pd[1].grad.double().cpu(), dba), "dqv": (pd[2].grad.double().cpu(), dqv)}


def _row_rel(a, b):
    """worst row of ||a - b|| / ||b|| (rows of b that are ~0 are measured against the matrix scale)"""
    scale = b.norm(dim=1).clamp_min(1e-3 * b.norm() / b.shape[0] ** 0.5)
    return float(((a - b).norm(dim=1) / scale).max())


def _rel(a, b):
    return float((a - b).norm() / b.norm())


SHAPES = [
    dict(N=3000, S=20, D=300, q=200),   # NRMS news level
    dict(N=512, S=50, D=300, q=200),    # user level
    dict(N=2000, S=3, D=300, q=200),    # Exp1 final attention
    dict(N=37, S=20, D=300, q=200),     # 740 rows: the last tile is partial
    dict(N=1, S=20, D=300, q=200),      # a single partial tile
    dict(N=300, S=20, D=300, q=24),     # q < 32: dPre leaves by plain stores
    dict(N=300, S=20, D=300, q=100),    # q % 16 != 0, the last dPre chunk cut by the query width
    dict(N=300, S=20, D=64, q=200),
    dict(N=300, S=20, D=320, q=200),
    dict(N=300, S=20, D=296, q=200),    # the last dX chunk of the second slice is cut
    dict(N=200, S=50, D=400, q=200),    # two weight slices of the input-gradient GEMM
]


@pytest.mark.parametrize("kw", SHAPES, ids=lambda kw: "N{N}_S{S}_D{D}_q{q}".format(**kw))
def test_additive_attention_bwd_rows_vs_fp64(kw):
    r = _run(seed=7, **kw)
    err = {"dx_rows": _row_rel(*r["dx"]), "dWa_rows": _row_rel(*r["dWa"]), "dba": _rel(*r["dba"]), "dqv": _rel(*r["dqv"])}
    # dX: one bf16 rounding of the stored row (2^-9 relative) on top of dPre elements one bf16 step away
    assert err["dx_rows"] < 8e-3, err
    assert err["dWa_rows"] < 5e-3 and err["dba"] < 5e-3, err
    assert err["dqv"] < 1e-3, err
