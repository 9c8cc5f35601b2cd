"""The additive-attention pooling forward (nr_additive_attention_fwd and its hi/lo form: pre = X . Wa^T on the wgmma GEMM,
then EpiPool's tanh scores, segment softmax and weighted row sum) judged element by element: every pooled output and every
saved softmax weight against an fp64 evaluation of the kernel's own bf16 X, Wa and fp32 ba, qv, with the error bound carried
stage by stage through the GEMM, tanh, the score, the softmax and the weighted sum (gpu_checks.additive_fwd_judge).

Cases (tests/gemm_cases.py POOL_CASES): every segment length class from 1 to 64, query widths below one 32-column chunk and
a streamed weight slice (D = 400, q = 200: NAML's pooling at F = 400), partial last tiles, one segment, more tiles than
CTAs, hi/lo planes split from fp32 rows, three score regimes (unit; peaked over +-100, which overflows fp32 without the max
subtraction; tied rows with exactly uniform weights) and an output pitch of 2 mod 4 (the scalar store path).  Around the
values: NaN in the pitch columns of X, X_lo and Wa never reaches an output, out's pitch columns and the guard bands keep
their pre-fill, a second run is bit-identical, and bad shapes are refused before any launch."""
import pytest
import torch

import gemm_cases as C
import gpu_checks as G

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _inputs(c, seed=3):
    """fp32 rows x [rows][D], Wa [q][D] (bf16 values), ba, qv [q] in the case's score regime."""
    n_seg, seg, D, q = c["n_seg"], c["seg"], c["D"], c["q"]
    rows = n_seg * seg
    g = torch.Generator().manual_seed(seed)
    x = torch.rand((rows, D), generator=g) * 2 - 1
    wa = (torch.rand((q, D), generator=g) * 2 - 1) * (3.0 / D) ** 0.5
    ba = (torch.rand((q,), generator=g) - 0.5) * 0.2
    qv = (torch.rand((q,), generator=g) * 2 - 1) * (3.0 / q) ** 0.5
    scores = c.get("scores", "unit")
    if scores == "peaked":  # column 0 drives every pre-activation into tanh saturation: score_r ~ 100 tanh(8 x_r0)
        wa[:, 1:] *= 0.1
        wa[:, 0] = 8.0
        qv = torch.full((q,), 100.0 / q)
    elif scores == "tied":  # every row of a segment equals its first
        x = x.view(n_seg, seg, D)[:, :1].expand(n_seg, seg, D).reshape(rows, D).clone()
    if not c.get("hilo"):
        x = x.to(torch.bfloat16).float()
    return x, wa.to(torch.bfloat16).float(), ba, qv


def _pack(c, x, wa, ba, qv):
    """Kernel operands: X (and X_lo) bf16 [rows][ldx] and Wa bf16 [q][ldx] with NaN in the pitch columns [D, ldx)."""
    D = c["D"]
    ldx = G.ru8(D + 1)
    X = torch.full((x.shape[0], ldx), float("nan"), dtype=torch.bfloat16, device=DEV)
    xd = x.to(DEV)
    X[:, :D] = xd.to(torch.bfloat16)
    X_lo = None
    if c.get("hilo"):
        X_lo = torch.full_like(X, float("nan"))
        X_lo[:, :D] = (xd - X[:, :D].float()).to(torch.bfloat16)
    Wa = torch.full((wa.shape[0], ldx), float("nan"), dtype=torch.bfloat16, device=DEV)
    Wa[:, :D] = wa.to(DEV).to(torch.bfloat16)
    return X, X_lo, Wa, ba.to(DEV), qv.to(DEV), ldx


def _launch(lib, c, X, X_lo, Wa, ba, qv, ldx, out_ptr, ldo, w_ptr, n_seg=None, seg=None, D=None, q=None):
    n_seg = c["n_seg"] if n_seg is None else n_seg
    seg = c["seg"] if seg is None else seg
    D = c["D"] if D is None else D
    q = c["q"] if q is None else q
    if X_lo is not None:
        return lib.nr_additive_attention_fwd_hilo(G._p(X), G._p(X_lo), n_seg, seg, D, ldx, G._p(Wa), q, ldx, G._p(ba), G._p(qv),
                                                  out_ptr, ldo, w_ptr, G._stream())
    return lib.nr_additive_attention_fwd(G._p(X), n_seg, seg, D, ldx, G._p(Wa), q, ldx, G._p(ba), G._p(qv), out_ptr, ldo, w_ptr,
                                         G._stream())


@pytest.mark.parametrize("c", C.POOL_CASES, ids=lambda c: c["id"])
def test_additive_fwd_elements(c):
    lib = G.load_library()
    n_seg, seg, D = c["n_seg"], c["seg"], c["D"]
    rows = n_seg * seg
    ldo = c.get("ldo", (D + 3) // 4 * 4 + 4)
    X, X_lo, Wa, ba, qv, ldx = _pack(c, *_inputs(c))
    runs = []
    for _ in range(2):
        out = G._Guarded(n_seg * ldo, torch.float32, float("nan"))
        out.prefill = out.body.clone()
        w = G._Guarded(rows, torch.float32, float("nan")) if c.get("w_out", True) else None
        G.check(_launch(lib, c, X, X_lo, Wa, ba, qv, ldx, G._p(out.all), ldo, G._p(w.all) if w is not None else None),
                "additive_attention_fwd")
        torch.cuda.synchronize()
        runs.append((out, w))
    out, w = runs[0]
    o = out.body.view(n_seg, ldo)[:, :D]
    j = G.additive_fwd_judge(X[:, :D].double(), Wa[:, :D].double(), ba.double(), qv.double(), seg, o,
                             w.body if w is not None else None, X_lo[:, :D].double() if X_lo is not None else None)
    pitch = torch.zeros(n_seg, ldo, dtype=torch.bool, device=DEV)
    pitch[:, D:] = True
    res = dict(j, pitch_untouched=out.unchanged(pitch), guards=all(b.guard_ok() for r in runs for b in r if b is not None),
               rerun_bit_identical=all(G._bits_equal(a.body, b.body) for a, b in zip(runs[0], runs[1]) if a is not None))
    assert res["out_ratio"] <= 1 and res.get("w_ratio", 0.0) <= 1, res
    assert res["pitch_untouched"] and res["guards"] and res["rerun_bit_identical"], res
    if c.get("scores") == "tied":  # equal rows give bit-equal scores: every weight is 1 / seg up to the division's rounding
        assert float((w.body - 1.0 / seg).abs().max()) <= 4 * G.U32, res
    print(c["id"], res)


def test_additive_fwd_refuses_bad_shapes_before_any_launch():
    """seg_len 0 or 65, q 0 or 257, odd D and odd output pitch are refused (seg_len 0 even though it makes no rows at all);
    n_seg = 0 is an empty problem that launches nothing."""
    lib = G.load_library()
    c = dict(n_seg=4, seg=8, D=64, q=32)
    X, _, Wa, ba, qv, ldx = _pack(c, *_inputs(c))
    Wa_big = torch.zeros(300, ldx, dtype=torch.bfloat16, device=DEV)
    qv_big = torch.zeros(300, device=DEV)
    out = G._Guarded(4 * 64, torch.float32, float("nan"))
    out.prefill = out.body.clone()
    n0 = lib.nr_launch_count()
    bad = [dict(seg=0), dict(seg=65, n_seg=1), dict(q=0), dict(q=257), dict(D=63), dict(ldo=63)]
    for b in bad:
        ldo = b.pop("ldo", 64)
        rc = _launch(lib, c, X, None, Wa_big, qv_big, qv_big, ldx, G._p(out.all), ldo, None, **b)
        assert rc != 0, b
    assert _launch(lib, c, X, None, Wa, ba, qv, ldx, G._p(out.all), 64, None, n_seg=0) == 0
    torch.cuda.synchronize()
    assert lib.nr_launch_count() == n0
    assert out.unchanged(torch.ones(out.n, dtype=torch.bool, device=DEV)) and out.guard_ok()
