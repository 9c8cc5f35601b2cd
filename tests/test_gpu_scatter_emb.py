"""The embedding-gradient scatter (gemm_scatter_emb: dEmb[ids[r]] += dY_r . W) at the edges of its live-tile list, through
nr_element_encoder_bwd, which takes any N (= E), K (= F) and ids.  The scatter processes only the 64-row tiles that hold a
row with an id in [1, V), so these cases place the live rows at tile edges, leave long dead runs, a live partial last tile,
fewer live tiles than CTAs and none at all.  Every case judges dEmb row by row against an fp64 reference from the same bf16
operands; the rows no valid id points at (row 0 among them) must keep their pre-fill bit for bit, and the guards behind the
buffers must be intact.  The encoders' own tests cover dropout and the row-mapped CNN layout through the same kernel."""
import math

import pytest
import torch

import gpu_checks as G
import newsrec_oracle as O
from newsrec_b200 import check, load_library
from newsrec_b200.ops import _p, _stream, cast_pad, ru8

pytestmark = pytest.mark.gpu


def run_scatter(ids, E, F, V, seed=7):
    """dY = bf16(dout) (out > 0 everywhere: no ReLU mask), then the scatter; returns the checks of dtable."""
    lib = load_library()
    n = ids.numel()
    lde, ldf = ru8(E + 1), ru8(F + 1)
    ids = ids.to(G.DEV)
    W = G._rand_bf16((F, E), seed, math.sqrt(3.0 / E)).to(G.DEV)
    wT = cast_pad(W, ldf, transpose=True)
    Eb = cast_pad(G._rand_bf16((n, E), seed + 1).to(G.DEV), lde)
    out = torch.ones(n, F, device=G.DEV)
    dout = O.det_uniform((n, F), seed + 2).to(G.DEV)
    dY = G._Guarded(n * ldf, torch.bfloat16, float("nan"))
    dW = G._Guarded(F * lde, torch.float32, 0.0)
    pat = O.det_uniform((V * E,), seed + 3, 0.5, 1.0).to(G.DEV) * 2.0 ** -16
    dt = G._Guarded(V * E, torch.float32, pat)
    check(lib.nr_element_encoder_bwd(_p(ids), n, _p(dout), _p(out), F, _p(dY.all), ldf, _p(Eb), E, lde, _p(wT), _p(dW.all),
                                     _p(dt.all), V, _stream()), "nr_element_encoder_bwd")
    torch.cuda.synchronize()
    dy64 = dY.body.view(n, ldf)[:, :F].double()
    live = (ids >= 1) & (ids < V)
    touched = torch.zeros(V, dtype=torch.bool, device=G.DEV)
    touched[ids[live]] = True
    res = {"guards_intact": dY.guard_ok() and dW.guard_ok() and dt.guard_ok(), "dev_error": G._dev_error(lib)[0],
           "untouched_rows_exact": dt.unchanged(~touched[:, None].expand(V, E)), "touched_rows": int(touched.sum())}
    if res["touched_rows"]:
        ref = torch.zeros(V, E, dtype=torch.float64, device=G.DEV).index_add_(0, ids[live], dy64[live] @ W.double())
        absref = torch.zeros(V, E, dtype=torch.float64, device=G.DEV).index_add_(0, ids[live], dy64[live].abs() @ W.double().abs())
        got = dt.body.view(V, E).double() - dt.prefill.view(V, E).double()
        res["row_ratio"] = G._abs_allow_rows(got[touched], ref[touched], absref[touched])
    return res


def assert_scatter(r, touched):
    assert r["guards_intact"] and r["dev_error"] == 0 and r["untouched_rows_exact"], r
    assert r["touched_rows"] == touched, r
    if touched:
        assert r["row_ratio"] <= 2e-6, r


def ids_with(n, live_rows, V):
    """n padding ids, with distinct valid ids (spread over [1, V)) at live_rows"""
    assert len(live_rows) < V
    ids = torch.zeros(n, dtype=torch.int64)
    ids[torch.tensor(live_rows, dtype=torch.int64)] = V - 1 - torch.arange(len(live_rows)) * ((V - 1) // len(live_rows))
    return ids


def test_all_tiles_dead():
    """Padding, negative and out-of-range ids only: no tile is live, every CTA leaves at once and dtable keeps its pre-fill."""
    ids = torch.zeros(64 * 300 + 5, dtype=torch.int64)
    ids[::7], ids[3::11] = -1, 500
    assert_scatter(run_scatter(ids, E=300, F=912, V=500), 0)


@pytest.mark.parametrize("row", [0, 63, 64, 127, 128, 64 * 150 - 1, 64 * 150, 64 * 300 + 4])
def test_one_live_row(row):
    """One live row at the first and last row of a tile and across tile edges, in a batch with a partial last tile."""
    n = 64 * 300 + 5
    ids = torch.zeros(n, dtype=torch.int64)
    ids[row] = 17
    assert_scatter(run_scatter(ids, E=300, F=912, V=500), 1)


def test_dead_runs_longer_than_the_grid():
    """Live tiles thousands of tiles apart (runs of dead tiles far longer than the grid's few dozen tile groups)."""
    n = 64 * 9000
    rows = [5, 64 * 2500 + 63, 64 * 2501, 64 * 7000 + 31, n - 1]
    assert_scatter(run_scatter(ids_with(n, rows, V=4000), E=300, F=912, V=4000), len(rows))


def test_fewer_live_tiles_than_ctas():
    """Three tiles in all: most CTAs get no tile, the others one each on one warpgroup."""
    n = 64 * 3 - 10
    assert_scatter(run_scatter(ids_with(n, list(range(n)), V=100000), E=300, F=912, V=100000), n)


def test_live_partial_last_tile():
    n = 64 * 40 + 17
    rows = list(range(64 * 40, n))
    assert_scatter(run_scatter(ids_with(n, rows, V=5000), E=300, F=912, V=5000), len(rows))


def test_mixed_ids_bench_like():
    """Left-padded histories and right-padded titles in impression-major order (55 news x 20 tokens, histories of 50 news
    padded on the left with all-zero news), plus negative and out-of-range ids, at N = 300, K = 912."""
    B, H, C, T, V = 96, 50, 5, 20, 7000
    g = torch.Generator().manual_seed(11)
    hist = torch.zeros(B, H, T, dtype=torch.int64)
    cand = torch.zeros(B, C, T, dtype=torch.int64)
    for b in range(B):
        n_hist = int(torch.randint(0, H + 1, (1,), generator=g))
        for h in range(H - n_hist, H):
            length = int(torch.randint(1, T + 1, (1,), generator=g))
            hist[b, h, :length] = torch.randint(1, V, (length,), generator=g)
        for c in range(C):
            length = int(torch.randint(1, T + 1, (1,), generator=g))
            cand[b, c, :length] = torch.randint(1, V, (length,), generator=g)
    ids = torch.cat([hist.reshape(-1), cand.reshape(-1)])
    ids[1234], ids[-3] = -5, V + 2
    live = (ids >= 1) & (ids < V)
    assert_scatter(run_scatter(ids, E=300, F=912, V=V), int(torch.unique(ids[live]).numel()))


@pytest.mark.parametrize("E,F", [(100, 400), (4, 8), (296, 64), (300, 300)])
def test_widths_and_heavy_repetition(E, F):
    """Every id repeats hundreds of times; N from one 4-column group to a partial last 32-column chunk."""
    n = 64 * 200 + 33
    ids = O.det_randint((n,), 5, 0, 6)
    assert_scatter(run_scatter(ids, E=E, F=F, V=6), 5)
