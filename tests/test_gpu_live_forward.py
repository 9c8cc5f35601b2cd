"""The NRMS news encoder's forward over live tokens (nr_mhsa_encoder_fwd_args.live).  A token is live when its id is in [1, V),
or when row 0 of the bf16 table is nonzero (then every token is).  With `live` the forward classifies the tokens once, gathers
and projects the live tokens' rows only, in compact order, and the title attention reads a dead token's Q|K|V from the bias
rows; the backward reuses the compaction, the compact X and the compact Q|K|V.

Every case runs twice on the same inputs, with `live` and without it:
- forward: out, w and both context planes are the same bits; compact row i of X, Q|K|V and V_lo is the same bits as row
  index[i] of the full run, and the rows behind the live ones up to the next 64-row tile are finite; the bad-id flag agrees;
- backward: the Q|K|V weight gradient, its bias column and the embedding gradient (rows 0 and 1 aside) agree to the fp32
  summation order, the pooling gradients within their run-to-run spread;
- refusals: `live` on the dense variant and at a shape the title kernels do not take returns -1 before any launch."""
import ctypes as C

import pytest
import torch

import gpu_checks as G
import newsrec_oracle as O
import test_gpu_live_tokens as L
import test_gpu_padding_news as P
from newsrec_b200 import MhsaEncoderBwdArgs, MhsaEncoderFwdArgs, check, launch_count, load_library
from newsrec_b200.ops import _p, _stream, qkv_pitches, ru8, ru16

pytestmark = pytest.mark.gpu
DEV = G.DEV
T, D, HEADS, Q, V = P.T, P.D, P.HEADS, P.Q, P.V


def _bench_ids(seed):
    """One bench batch of NRMS titles (bench.synth_slots: 512 impressions x 55 news, right-padded titles, left-padded
    histories), its word ids folded into [1, V)."""
    import bench
    _, cand, hist = bench.synth_slots("NRMS", 512, seed)
    ids = torch.stack([s["title"] for s in cand + hist], 1).reshape(-1, T)
    ids = torch.where(ids > 0, (ids - 1) % (V - 1) + 1, ids)
    return ids.shape[0], ids.reshape(-1).contiguous()


def _ids(name, seed):
    return _bench_ids(seed) if name == "bench" else L._ids(name, seed)


def _run(ids, ops, n_seq, seed, live, accurate, p_drop=0.2):
    lib = load_library()
    ldx, ldq = ru8(D + 1), ru16(Q)
    sec, ld3 = qkv_pitches(D)
    n_tok = n_seq * T
    nan = float("nan")
    f = dict(X=torch.full((n_tok, ldx), nan, dtype=torch.bfloat16, device=DEV),
             QKV=torch.full((n_tok, ld3), nan, dtype=torch.bfloat16, device=DEV),
             Vlo=torch.full((n_tok, sec), nan, dtype=torch.bfloat16, device=DEV),
             C=torch.full((n_tok, ldx), nan, dtype=torch.bfloat16, device=DEV),
             Clo=torch.full((n_tok, ldx), nan, dtype=torch.bfloat16, device=DEV),
             w=torch.full((n_tok,), nan, device=DEV), out=torch.full((n_seq, D), nan, device=DEV),
             flag=torch.zeros(1, dtype=torch.int32, device=DEV))
    a = MhsaEncoderFwdArgs()
    a.n_seq, a.T, a.d, a.heads, a.q, a.ldx, a.ld3 = n_seq, T, D, HEADS, Q, ldx, ld3
    a.ids, a.table_bf16, a.V = _p(ids), _p(ops["table"]), V
    a.wqkv_bf16, a.bqkv, a.wa_bf16, a.ba, a.qv = _p(ops["wqkv"]), _p(ops["bqkv"]), _p(ops["wa"]), _p(ops["ba"]), _p(ops["qv"])
    a.p_drop, a.seed = p_drop, 0x5EED + seed
    a.X_bf16, a.QKV_bf16, a.C_bf16, a.w, a.out = _p(f["X"]), _p(f["QKV"]), _p(f["C"]), _p(f["w"]), _p(f["out"])
    a.bad_id_flag = _p(f["flag"])
    if accurate:
        a.V_lo_bf16, a.C_lo_bf16 = _p(f["Vlo"]), _p(f["Clo"])
    buf = None
    if live:
        nb = int(lib.nr_mhsa_encoder_live_bytes(n_seq, T, D))
        buf = torch.full((nb,), 0xFF, dtype=torch.uint8, device=DEV)
        a.live, a.live_bytes = _p(buf), nb
    check(lib.nr_mhsa_encoder_fwd(C.byref(a), _stream()), "nr_mhsa_encoder_fwd")

    dout = O.det_uniform((n_seq, D), seed + 14).to(DEV)
    g = dict(dW3=torch.zeros((3 * sec, ldx), device=DEV), dWa=torch.zeros((Q, ldx), device=DEV), dqv=torch.zeros(Q, device=DEV),
             demb=torch.zeros((V, D), device=DEV))
    ws_bytes = int(lib.nr_mhsa_encoder_bwd_workspace(n_seq, T, D, Q))
    ws = torch.full((ws_bytes,), 0xFF, dtype=torch.uint8, device=DEV)
    b = MhsaEncoderBwdArgs()
    b.n_seq, b.T, b.d, b.heads, b.q, b.ldx, b.ld3, b.ldq = n_seq, T, D, HEADS, Q, ldx, ld3, ldq
    b.ids, b.V, b.table_bf16 = _p(ids), V, _p(ops["table"])
    b.wqkvT_bf16, b.wa_bf16, b.waT_bf16, b.ba, b.qv = _p(ops["wqkvT"]), _p(ops["wa"]), _p(ops["waT"]), _p(ops["ba"]), _p(ops["qv"])
    b.p_drop, b.seed = p_drop, 0x5EED + seed
    b.X_bf16, b.QKV_bf16, b.C_bf16, b.w, b.dout = _p(f["X"]), _p(f["QKV"]), _p(f["C"]), _p(f["w"]), _p(dout)
    b.wqkv_bf16, b.bqkv = _p(ops["wqkv"]), _p(ops["bqkv"])
    b.dWqkv_ext, b.dWa_ext, b.dqv, b.demb = _p(g["dW3"]), _p(g["dWa"]), _p(g["dqv"]), _p(g["demb"])
    b.workspace, b.workspace_bytes = _p(ws), ws_bytes
    if live:
        b.live, b.live_bytes = _p(buf), buf.numel()
    check(lib.nr_mhsa_encoder_bwd(C.byref(b), _stream()), "nr_mhsa_encoder_bwd")
    torch.cuda.synchronize()
    return f, g


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


@pytest.mark.parametrize("accurate", [True, False])
@pytest.mark.parametrize("row0_zero", [True, False])
@pytest.mark.parametrize("name", L.NAMES + ["bench"])
def test_live_forward_matches_full(name, row0_zero, accurate):
    seed = 7 + len(name)
    n_seq, ids = _ids(name, seed)
    ids = ids.to(DEV)
    ops = P._operands(seed, row0_zero)
    fc, gc = _run(ids, ops, n_seq, seed, live=True, accurate=accurate)
    ff, gf = _run(ids, ops, n_seq, seed, live=False, accurate=accurate)
    planes = ("out", "w", "C") + (("Clo",) if accurate else ())
    for k in planes:
        assert not torch.isnan(ff[k].float()).any(), k
        assert torch.equal(_bits(fc[k]), _bits(ff[k])), k
    assert int(fc["flag"]) == int(ff["flag"])
    # the compact rows against the full run's rows of their tokens
    e = L._expected(ids, n_seq, None, ru8(D + 1), not row0_zero, True)
    m, index = e["m_live"], e["index"].to(DEV)
    M = n_seq * T
    tail = min(M, (m + 63) // 64 * 64)
    for k in ("X", "QKV") + (("Vlo",) if accurate else ()):
        assert torch.equal(_bits(fc[k][:m]), _bits(ff[k][index])), k
    assert bool((fc["X"][m:tail].float() == 0).all())
    assert torch.isfinite(fc["QKV"][m:tail].float()).all()
    gc["demb"][:2] = 0
    gf["demb"][:2] = 0
    parts = dict(dW3=(gc["dW3"][:, :D], gf["dW3"][:, :D]), dW3_bias=(gc["dW3"][:, D], gf["dW3"][:, D]), demb=(gc["demb"], gf["demb"]),
                 dWa=(gc["dWa"], gf["dWa"]), dqv=(gc["dqv"], gf["dqv"]))
    for k, (x, y) in parts.items():
        assert torch.isfinite(x).all(), k
        err, tol = float((x - y).abs().max()), 1e-5 * float(y.abs().max()) + 1e-30
        assert err <= tol, (k, err, tol)


@pytest.mark.parametrize("case", ["dense", "non_title_shape"])
def test_live_refused_outside_the_title_kernels(case):
    lib = load_library()
    n_seq, Tn, d, heads = (4, T, D, HEADS) if case == "dense" else (4, 16, 64, 4)
    ldx = ru8(d + 1)
    sec, ld3 = qkv_pitches(d)
    n_tok = n_seq * Tn
    bf = lambda *s: torch.zeros(s, dtype=torch.bfloat16, device=DEV)  # noqa: E731
    keep = dict(X=bf(n_tok, ldx), QKV=bf(n_tok, ld3), C=bf(n_tok, ldx), wqkv=bf(3 * sec, ldx), wa=bf(Q, ldx), table=bf(V, ldx),
                bqkv=torch.zeros(3 * sec, device=DEV), ba=torch.zeros(Q, device=DEV), qv=torch.zeros(Q, device=DEV),
                w=torch.zeros(n_tok, device=DEV), out=torch.zeros((n_seq, d), device=DEV), flag=torch.zeros(1, dtype=torch.int32, device=DEV),
                ids=torch.ones(n_tok, dtype=torch.long, device=DEV), dense=torch.zeros((n_seq, Tn, d), device=DEV))
    nb = int(lib.nr_mhsa_encoder_live_bytes(n_seq, Tn, d))
    buf = torch.zeros(nb, dtype=torch.uint8, device=DEV)
    a = MhsaEncoderFwdArgs()
    a.n_seq, a.T, a.d, a.heads, a.q, a.ldx, a.ld3 = n_seq, Tn, d, heads, Q, ldx, ld3
    if case == "dense":
        a.dense = _p(keep["dense"])
        a.dense_s_seq, a.dense_s_tok, a.dense_s_col = keep["dense"].stride()
    else:
        a.ids, a.table_bf16, a.V = _p(keep["ids"]), _p(keep["table"]), V
    a.wqkv_bf16, a.bqkv, a.wa_bf16, a.ba, a.qv = _p(keep["wqkv"]), _p(keep["bqkv"]), _p(keep["wa"]), _p(keep["ba"]), _p(keep["qv"])
    a.X_bf16, a.QKV_bf16, a.C_bf16, a.w, a.out, a.bad_id_flag = (_p(keep[k]) for k in ("X", "QKV", "C", "w", "out", "flag"))
    a.live, a.live_bytes = _p(buf), nb
    torch.cuda.synchronize()
    l0 = launch_count()
    assert lib.nr_mhsa_encoder_fwd(C.byref(a), _stream()) == -1
    assert launch_count() == l0

    ws_bytes = int(lib.nr_mhsa_encoder_bwd_workspace(n_seq, Tn, d, Q))
    ws = torch.zeros(ws_bytes, dtype=torch.uint8, device=DEV)
    b = MhsaEncoderBwdArgs()
    b.n_seq, b.T, b.d, b.heads, b.q, b.ldx, b.ld3, b.ldq = n_seq, Tn, d, heads, Q, ldx, ld3, ru16(Q)
    dW3, dWa, dqv = torch.zeros((3 * sec, ldx), device=DEV), torch.zeros((Q, ldx), device=DEV), torch.zeros(Q, device=DEV)
    demb, ddense = torch.zeros((V, d), device=DEV), torch.zeros((n_tok, d), device=DEV)
    if case == "dense":
        b.ddense = _p(ddense)
    else:
        b.ids, b.V, b.table_bf16, b.demb = _p(keep["ids"]), V, _p(keep["table"]), _p(demb)
    b.wqkvT_bf16, b.wa_bf16, b.waT_bf16, b.ba, b.qv = _p(keep["wqkv"]), _p(keep["wa"]), _p(keep["wa"]), _p(keep["ba"]), _p(keep["qv"])
    b.X_bf16, b.QKV_bf16, b.C_bf16, b.w, b.dout = _p(keep["X"]), _p(keep["QKV"]), _p(keep["C"]), _p(keep["w"]), _p(keep["out"])
    b.bqkv = _p(keep["bqkv"])
    b.dWqkv_ext, b.dWa_ext, b.dqv = _p(dW3), _p(dWa), _p(dqv)
    b.workspace, b.workspace_bytes = _p(ws), ws_bytes
    b.live, b.live_bytes = _p(buf), nb
    l0 = launch_count()
    assert lib.nr_mhsa_encoder_bwd(C.byref(b), _stream()) == -1
    assert launch_count() == l0
