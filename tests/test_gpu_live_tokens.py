"""The backward of the accurate NRMS news encoder over live tokens only.  A token is live when its id is in [1, V), or when row 0
of the bf16 table is nonzero (then every token is).  A dead token's gathered row is [0 .. 0, 1], so its dQ|dK|dV row adds
nothing to the embedding gradient and reaches the Q|K|V weight gradient only through the bias column.  The backward stores the
live tokens' dQ|dK|dV rows in compact order, sums the dead tokens' rows into the bias column inside the title attention, and
runs the embedding scatter and the weight-gradient GEMM over the compact rows.

Two checks per pattern:
- the compaction on its own (nr_debug_live_tokens) against a restatement in Python: live masks, padding flags, offsets, the
  compact -> token index, the tile list, the compact copy of X and the zero tail rows, with the table and without it (then
  the verdict comes from the gathered rows);
- the whole backward against a stand-in run: every id 0 becomes id 1, whose table row is row 0's copy, so the gathered rows
  are the same bits but nothing is compacted away.  The forward's outputs must be the same bits; the Q|K|V weight gradient,
  its bias, the pooling gradients and every embedding-gradient row but rows 0 and 1 must agree to the fp32 summation
  order."""
import ctypes as C

import pytest
import torch

import gpu_checks as G
import newsrec_oracle as O
import test_gpu_padding_news as P
from newsrec_b200 import MhsaEncoderBwdArgs, MhsaEncoderFwdArgs, check, load_library
from newsrec_b200.ops import _p, _stream, qkv_pitches, ru8, ru16

pytestmark = pytest.mark.gpu
DEV = G.DEV
T, D, HEADS, Q, V = P.T, P.D, P.HEADS, P.Q, P.V


def _ids(name, seed):
    """(n_seq, ids [n_seq * T]) of one pattern."""
    gen = torch.Generator().manual_seed(seed)
    if name == "all_live":          # 32 titles of 20 real words: M' = 640, ten whole tiles
        n_seq = 32
        ids = torch.randint(2, V, (n_seq, T), generator=gen)
    elif name == "all_dead":
        n_seq = 24
        ids = torch.zeros((n_seq, T), dtype=torch.long)
    elif name == "padding_titles":  # left-padded histories: runs of all-zero titles between real ones
        n_seq = 120
        ids = torch.randint(2, V, (n_seq, T), generator=gen)
        ids[:, 15:] = 0
        ids[3:60] = 0
        ids[70:117] = 0
    elif name == "zeros_inside":    # unknown words map to 0 inside a title, right padding after it
        n_seq = 40
        ids = torch.randint(2, V, (n_seq, T), generator=gen)
        ids[torch.rand((n_seq, T), generator=gen) < 0.3] = 0
        ids[:, 17:] = 0
    elif name == "out_of_range":    # read as row 0 by the gather (which raises its flag), dead like id 0
        n_seq = 30
        ids = torch.randint(2, V, (n_seq, T), generator=gen)
        ids[:, 12:] = 0
        ids[4, 3], ids[9, 0], ids[17, 11] = V + 3, -1, V
        ids[22] = V + 7
    elif name == "multiple_of_64":  # 16 live tokens per title: M' = 16 * 16 = 256
        n_seq = 16
        ids = torch.randint(2, V, (n_seq, T), generator=gen)
        ids[:, 16:] = 0
    elif name == "partial_last":    # 15 live tokens per title: M' = 555, a last compact tile of 43 rows
        n_seq = 37
        ids = torch.randint(2, V, (n_seq, T), generator=gen)
        ids[:, 15:] = 0
    else:
        raise KeyError(name)
    return n_seq, ids.reshape(-1).contiguous()


NAMES = ["all_live", "all_dead", "padding_titles", "zeros_inside", "out_of_range", "multiple_of_64", "partial_last"]


def _expected(ids, n_seq, X, ldx, row0_nonzero, use_table):
    """The compaction restated on the host."""
    ids = ids.cpu().view(n_seq, T)
    live = (ids >= 1) & (ids < V)
    if use_table:
        if row0_nonzero:
            live[:] = True
    else:
        live |= ((X.cpu().view(torch.int16)[:, :D] & 0x7FFF) != 0).any(1).view(n_seq, T)
    mask = (live.long() << torch.arange(T)).sum(1)
    counts = live.sum(1)
    offset = torch.zeros(n_seq + 1, dtype=torch.long)
    offset[1:] = torch.cumsum(counts, 0)
    index = torch.nonzero(live.reshape(-1)).reshape(-1)
    m_live = int(offset[-1])
    return dict(mask=mask, pad=(counts == 0).long(), offset=offset, index=index, m_live=m_live, tiles=(m_live + 63) // 64)


@pytest.mark.parametrize("use_table", [True, False])
@pytest.mark.parametrize("row0_zero", [True, False])
@pytest.mark.parametrize("name", NAMES)
def test_live_token_compaction_matches_host(name, row0_zero, use_table):
    lib = load_library()
    seed = 7 + len(name)
    n_seq, ids = _ids(name, seed)
    ops = P._operands(seed, row0_zero)
    ldx = ru8(D + 1)
    sec, ld3 = qkv_pitches(D)
    M = n_seq * T
    ids_d = ids.to(DEV)
    # X as the gather leaves it: the table row (row 0 for an out-of-range id), the ones column at D
    safe = torch.where((ids >= 0) & (ids < V), ids, torch.zeros_like(ids)).to(DEV)
    X = ops["table"][safe].clone()
    X[:, D] = 1.0
    out = dict(mask=torch.full((n_seq,), -1, dtype=torch.int32, device=DEV), pad=torch.full((n_seq,), 7, dtype=torch.uint8, device=DEV),
               offset=torch.full((n_seq + 1,), -7, dtype=torch.int32, device=DEV), index=torch.full((M,), -7, dtype=torch.int32, device=DEV),
               tiles=torch.full((1 + (M + 63) // 64,), -7, dtype=torch.int32, device=DEV),
               Xc=torch.full((M, ldx), float("nan"), dtype=torch.bfloat16, device=DEV),
               dq=torch.full((M, ld3), float("nan"), dtype=torch.bfloat16, device=DEV))
    check(lib.nr_debug_live_tokens(_p(ids_d), n_seq, T, D, _p(ops["table"]) if use_table else None, V, _p(X), ldx, _p(ops["bqkv"]),
                                   _p(out["mask"]), _p(out["pad"]), _p(out["offset"]), _p(out["index"]), _p(out["tiles"]),
                                   _p(out["Xc"]), _p(out["dq"]), _stream()), "nr_debug_live_tokens")
    torch.cuda.synchronize()
    e = _expected(ids, n_seq, X, ldx, not row0_zero, use_table)
    m = e["m_live"]
    assert torch.equal(out["mask"].cpu().long() & 0xFFFFF, e["mask"])
    assert torch.equal(out["pad"].cpu().long(), e["pad"])
    assert torch.equal(out["offset"].cpu().long(), e["offset"])
    assert torch.equal(out["index"][:m].cpu().long(), e["index"])
    tail = min(M, (m + 63) // 64 * 64)
    assert bool((out["index"][m:tail] == -1).all())
    tiles = out["tiles"].cpu().long()
    assert int(tiles[0]) == e["tiles"]
    assert torch.equal(tiles[1:1 + e["tiles"]], torch.arange(e["tiles"]))
    assert torch.equal(out["Xc"][:m].view(torch.int16), X[e["index"].to(DEV)].view(torch.int16))
    assert bool((out["Xc"][m:tail].float() == 0).all()) and bool((out["dq"][m:tail].float() == 0).all())


def _run(ids, ops, n_seq, seed, p_drop=0.2):
    """P._run with the forward's table passed to the backward as well."""
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
    a.bad_id_flag, a.V_lo_bf16, a.C_lo_bf16 = _p(f["flag"]), _p(f["Vlo"]), _p(f["Clo"])
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
    check(lib.nr_mhsa_encoder_bwd(C.byref(b), _stream()), "nr_mhsa_encoder_bwd")
    torch.cuda.synchronize()
    return f, g


@pytest.mark.parametrize("row0_zero", [True, False])
@pytest.mark.parametrize("name", NAMES)
def test_live_token_backward_matches_stand_in(name, row0_zero):
    seed = 7 + len(name)
    n_seq, ids = _ids(name, seed)
    ids = ids.to(DEV)
    stand_in = torch.where(ids == 0, torch.ones_like(ids), ids)
    ops = P._operands(seed, row0_zero)
    f1, g1 = _run(ids, ops, n_seq, seed)
    f2, g2 = _run(stand_in, ops, n_seq, seed)
    for k in ("out", "w", "C", "Clo"):
        assert not torch.isnan(f1[k].float()).any(), k
        assert torch.equal(f1[k].view(torch.int16) if f1[k].dtype == torch.bfloat16 else f1[k].view(torch.int32),
                           f2[k].view(torch.int16) if f2[k].dtype == torch.bfloat16 else f2[k].view(torch.int32)), k
    g1["demb"][:2] = 0
    g2["demb"][:2] = 0
    # the bias column on its own scale: leaving out one dead row of a title would move it far past the tolerance.  The pooling
    # gradients come before the projection backward, but their GEMM adds by atomics too: the same sums, in any order
    parts = dict(dW3=(g1["dW3"][:, :D], g2["dW3"][:, :D]), dW3_bias=(g1["dW3"][:, D], g2["dW3"][:, D]), demb=(g1["demb"], g2["demb"]),
                 dWa=(g1["dWa"], g2["dWa"]), dqv=(g1["dqv"], g2["dqv"]))
    for k, (x, y) in parts.items():
        assert torch.isfinite(x).all(), k
        err, tol = float((x - y).abs().max()), 1e-5 * float(y.abs().max()) + 1e-30
        assert err <= tol, (k, err, tol)
