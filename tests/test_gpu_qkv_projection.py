"""The news-level Q|K|V projection of the accurate NRMS encoder (nr_mhsa_encoder_fwd with a V low plane), element by element
against an fp64 evaluation of the same bf16 operands.  The projection's store epilogue writes Q|K|V in bf16 through TMA and,
for the V section, the low plane bf16(y - bf16(y)) through a second tensor map; the model-level golden cases see these only
through the pooled output.  Every "=" output starts as NaN and is followed by sentinel guards (gpu_checks._Guarded)."""
import ctypes as C
import math

import pytest
import torch

import gpu_checks as G
import newsrec_oracle as O
from newsrec_b200 import MhsaEncoderFwdArgs, check, load_library
from newsrec_b200.ops import _p, _stream, cast_pad, qkv_pitches, ru8, stack_qkv

pytestmark = pytest.mark.gpu
DEV = G.DEV


def check_qkv_projection(n_seq, T=20, d=300, heads=15, q=200, V=500, p_drop=0.2, accurate=True, seed=3):
    lib = load_library()
    ldx = ru8(d + 1)
    sec, ld3 = qkv_pitches(d)
    n_tok = n_seq * T
    a_w = math.sqrt(3.0 / d)
    Wq, Wk, Wv = (G._rand_bf16((d, d), seed + i, a_w).to(DEV) for i in range(3))
    bq, bk, bv = (O.det_uniform((d,), seed + 3 + i, -0.5, 0.5).to(DEV) for i in range(3))
    wqkv = cast_pad(stack_qkv(Wq, Wk, Wv), ldx)
    bqkv = stack_qkv(bq, bk, bv).contiguous()
    wa = cast_pad(G._rand_bf16((q, d), seed + 6, math.sqrt(3.0 / d)).to(DEV), ldx)
    ba = O.det_uniform((q,), seed + 7, -0.1, 0.1).to(DEV)
    qv = O.det_uniform((q,), seed + 8).to(DEV)
    table = cast_pad(G._rand_bf16((V, d), seed + 9).to(DEV), ldx)
    ids = O.synth_titles(n_seq, T, V, seed + 10).to(DEV)

    nan = float("nan")
    bufs = dict(X=G._Guarded(n_tok * ldx, torch.bfloat16, nan), QKV=G._Guarded(n_tok * ld3, torch.bfloat16, nan),
                C=G._Guarded(n_tok * ldx, torch.bfloat16, nan), w=G._Guarded(n_tok, torch.float32, nan),
                out=G._Guarded(n_seq * d, torch.float32, nan), flag=G._Guarded(1, torch.int32, 0, sentinel=-7))
    if accurate:
        bufs["Vlo"] = G._Guarded(n_tok * sec, torch.bfloat16, nan)
        bufs["Clo"] = G._Guarded(n_tok * ldx, torch.bfloat16, nan)
    a = MhsaEncoderFwdArgs()
    a.n_seq, a.T, a.d, a.heads, a.q, a.ldx, a.ld3 = n_seq, T, d, heads, q, ldx, ld3
    a.ids, a.table_bf16, a.V = _p(ids), _p(table), V
    a.wqkv_bf16, a.bqkv, a.wa_bf16, a.ba, a.qv = _p(wqkv), _p(bqkv), _p(wa), _p(ba), _p(qv)
    a.p_drop, a.seed = float(p_drop), 0x1234567 + seed
    a.X_bf16, a.QKV_bf16, a.C_bf16 = _p(bufs["X"].all), _p(bufs["QKV"].all), _p(bufs["C"].all)
    a.w, a.out, a.bad_id_flag = _p(bufs["w"].all), _p(bufs["out"].all), _p(bufs["flag"].all)
    if accurate:
        a.V_lo_bf16, a.C_lo_bf16 = _p(bufs["Vlo"].all), _p(bufs["Clo"].all)
    check(lib.nr_mhsa_encoder_fwd(C.byref(a), _stream()), "nr_mhsa_encoder_fwd")
    torch.cuda.synchronize()

    res = {"guards_intact": all(b.guard_ok() for b in bufs.values()), "hi_ratio": 0.0, "hilo_ratio": 0.0,
           "nonfinite": 0, "pad_nonzero": 0}
    X = bufs["X"].body.view(n_tok, ldx)
    QKV = bufs["QKV"].body.view(n_tok, ld3)
    Vlo = bufs["Vlo"].body.view(n_tok, sec) if accurate else None
    W64 = wqkv[:, :d].double()
    b64 = bqkv.double()
    pad_cols = torch.tensor([s * sec + c for s in range(3) for c in range(d, sec)], dtype=torch.long, device=DEV)
    for r0 in range(0, n_tok, 32768):  # fp64 temporaries of a few hundred MB per chunk
        r1 = min(n_tok, r0 + 32768)
        x = X[r0:r1, :d].double()
        ref = x @ W64.t() + b64
        absum = x.abs() @ W64.abs().t() + b64.abs()
        hi = QKV[r0:r1, :3 * sec].double()
        res["nonfinite"] += int((~torch.isfinite(hi)).sum())
        res["pad_nonzero"] += int((hi[:, pad_cols] != 0).sum())
        # one bf16 rounding of the fp32 result, plus the fp32 accumulation over K = 300
        bound = G._bf16_ulp(torch.maximum(ref.abs(), hi.abs())) + 1e-6 * absum
        res["hi_ratio"] = max(res["hi_ratio"], G._worst(G._safe_div((hi - ref).abs(), bound)))
        if accurate:
            lo = Vlo[r0:r1].double()
            res["nonfinite"] += int((~torch.isfinite(lo)).sum())
            res["pad_nonzero"] += int((lo[:, d:] != 0).sum())
            vref = ref[:, 2 * sec:3 * sec]
            err = (hi[:, 2 * sec:3 * sec] + lo - vref).norm(dim=1)
            rb = 2.0 ** -16 * vref.norm(dim=1) + 1e-6 * absum[:, 2 * sec:3 * sec].norm(dim=1)
            res["hilo_ratio"] = max(res["hilo_ratio"], G._worst(G._safe_div(err, rb)))
    return res


@pytest.mark.parametrize("kw", [
    dict(n_seq=28160),                  # the bench shape: batch 512 x (50 clicked + 5 candidate) titles, 563,200 tokens
    dict(n_seq=37),                     # 740 tokens: the last 64-row tile holds 36 rows
    dict(n_seq=37, accurate=False),     # fast mode: no low plane
])
def test_qkv_projection_matches_fp64(kw):
    r = check_qkv_projection(**kw)
    assert r["guards_intact"] and r["nonfinite"] == 0 and r["pad_nonzero"] == 0, r
    assert r["hi_ratio"] <= 1.0, r
    assert r["hilo_ratio"] <= 1.0, r
