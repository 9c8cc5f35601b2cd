"""The accurate NRMS news encoder (nr_mhsa_encoder_fwd / _bwd, ids variant) on batches with padding titles: all ids 0 and a
zero table row 0, the left-padding of short histories.  The encoder skips them: the projection computes only the live 64-row
tiles, the title attention reads their Q|K|V from one shared bias tile, and the weight gradient leaves out the tiles that hold
only padding rows and adds their dQ|dK|dV column sums to the bias column.

Each case runs the same batch twice.  In the second run every padding id 0 becomes id 1, whose table row is row 0's copy: the
gathered rows are the same bits, but no title is padding, so every stage does its full work.  Everything the forward writes
for the caller (news vectors, pooling weights, both context planes) must be the same bits; the gradients must agree to the
fp32 summation order (the weight gradients are accumulated by atomic adds in both runs), the embedding gradient outside rows
0 and 1 included.  The outputs start as NaN, so a row that either run leaves unwritten fails."""
import ctypes as C
import math

import pytest
import torch

import gpu_checks as G
import newsrec_oracle as O
from newsrec_b200 import MhsaEncoderBwdArgs, MhsaEncoderFwdArgs, check, load_library
from newsrec_b200.ops import _p, _stream, cast_pad, qkv_pitches, ru8, ru16, stack_qkv

pytestmark = pytest.mark.gpu
DEV = G.DEV
T, D, HEADS, Q, V = 20, 300, 15, 200, 500


def _operands(seed, row0_zero):
    a_w = 3.0 / math.sqrt(D)
    Wqkv = [G._rand_bf16((D, D), seed + 1 + i, a_w).to(DEV) for i in range(3)]
    bqkv = stack_qkv(*[O.det_uniform((D,), seed + 4 + i, -0.1, 0.1).to(DEV) for i in range(3)]).contiguous()
    Wa = G._rand_bf16((Q, D), seed + 7, math.sqrt(3.0 / D)).to(DEV)
    ldx, ldq = ru8(D + 1), ru16(Q)
    _, ld3 = qkv_pitches(D)
    wqkv_f = stack_qkv(*Wqkv)
    table = G._rand_bf16((V, D), seed + 10).to(DEV)
    if row0_zero:
        table[0] = 0
    table[1] = table[0]  # the stand-in id of the second run: the same row bits
    return dict(wqkv=cast_pad(wqkv_f, ldx), wqkvT=cast_pad(wqkv_f, ld3, transpose=True), bqkv=bqkv, wa=cast_pad(Wa, ldx),
                waT=cast_pad(Wa, ldq, transpose=True), ba=O.det_uniform((Q,), seed + 8, -0.1, 0.1).to(DEV),
                qv=O.det_uniform((Q,), seed + 9, -1.0, 1.0).to(DEV), table=cast_pad(table, ldx))


def _run(ids, ops, n_seq, seed, p_drop=0.2):
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
    b.ids, b.V = _p(ids), V
    b.wqkvT_bf16, b.wa_bf16, b.waT_bf16, b.ba, b.qv = _p(ops["wqkvT"]), _p(ops["wa"]), _p(ops["waT"]), _p(ops["ba"]), _p(ops["qv"])
    b.p_drop, b.seed = p_drop, 0x5EED + seed
    b.X_bf16, b.QKV_bf16, b.C_bf16, b.w, b.dout = _p(f["X"]), _p(f["QKV"]), _p(f["C"]), _p(f["w"]), _p(dout)
    b.wqkv_bf16, b.bqkv = _p(ops["wqkv"]), _p(ops["bqkv"])
    b.dWqkv_ext, b.dWa_ext, b.dqv, b.demb = _p(g["dW3"]), _p(g["dWa"]), _p(g["dqv"]), _p(g["demb"])
    b.workspace, b.workspace_bytes = _p(ws), ws_bytes
    check(lib.nr_mhsa_encoder_bwd(C.byref(b), _stream()), "nr_mhsa_encoder_bwd")
    torch.cuda.synchronize()
    return f, g


def _titles(pattern, n_seq, seed):
    """ids [n_seq][T] with the titles of `pattern` (a list of title indices, or a name) all 0."""
    gen = torch.Generator().manual_seed(seed)
    ids = torch.randint(2, V, (n_seq, T), generator=gen)
    ids[:, 15:] = 0  # right-padded words of real titles stay live
    pad = torch.zeros(n_seq, dtype=torch.bool)
    pad[pattern] = True
    ids[pad] = 0
    return ids


# 64-row tiles hold 3.2 titles: title s covers rows [20 s, 20 s + 20)
PATTERNS = {
    "none": (40, []),
    "all": (40, list(range(40))),
    "short_run": (40, [5, 6]),                              # 40 rows: no tile is all padding
    "history_runs": (120, list(range(3, 60)) + list(range(70, 117))),  # dead tiles between live ones, straddling titles
    "straddle": (40, list(range(4, 40))),                   # title 3 (rows 60..79) crosses the first tile edge and is live
    "inside_live": (48, [3] + list(range(7, 41))),          # title 3 is padding inside a live tile
    "dead_last_partial": (37, list(range(20, 37))),         # 740 rows: the last tile has 36 rows, all padding
    "one_token": (40, list(range(8, 40))),                  # plus title 20 below: zeros but one token
}


@pytest.mark.parametrize("row0_zero", [True, False])
@pytest.mark.parametrize("name", sorted(PATTERNS))
def test_padding_titles_match_full_work(name, row0_zero):
    n_seq, pattern = PATTERNS[name]
    seed = 3 + len(name)
    ids = _titles(pattern, n_seq, seed)
    if name == "one_token":
        ids[20, 7] = 11
    if name == "history_runs":
        ids[90, 4] = V + 3  # out of range: reads row 0 and raises the flag, and is not a padding title
    ids = ids.to(DEV).reshape(-1).contiguous()
    stand_in = torch.where(ids == 0, torch.ones_like(ids), ids)
    ops = _operands(seed, row0_zero)
    f1, g1 = _run(ids, ops, n_seq, seed)
    f2, g2 = _run(stand_in, ops, n_seq, seed)
    assert int(f1["flag"].item()) == int(f2["flag"].item()) == (1 if name == "history_runs" else 0)
    for k in ("out", "w", "C", "Clo"):
        assert not torch.isnan(f1[k].float()).any(), k
        assert torch.equal(f1[k].view(torch.int16) if f1[k].dtype == torch.bfloat16 else f1[k].view(torch.int32),
                           f2[k].view(torch.int16) if f2[k].dtype == torch.bfloat16 else f2[k].view(torch.int32)), k
    g1["demb"][:2] = 0
    g2["demb"][:2] = 0
    # the bias column of dWqkv on its own scale: leaving out one 64-row tile would move it by a few percent
    parts = dict(dW3=g1["dW3"][:, :D], dW3_bias=g1["dW3"][:, D], dWa=g1["dWa"], dqv=g1["dqv"], demb=g1["demb"])
    refs = dict(dW3=g2["dW3"][:, :D], dW3_bias=g2["dW3"][:, D], dWa=g2["dWa"], dqv=g2["dqv"], demb=g2["demb"])
    for k, x in parts.items():
        y = refs[k]
        assert torch.isfinite(x).all(), k
        err, tol = float((x - y).abs().max()), 1e-5 * float(y.abs().max()) + 1e-30
        assert err <= tol, (k, err, tol)
