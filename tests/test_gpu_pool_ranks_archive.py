"""Ranks over the whole pool under Hi-Fi Ark's and DKN's DNN click score on the H100: nr_pool_ranks_archive /
ops.pool_ranks(..., dnn=) exactly against nr_topk_archive's lists (the same score bits), within the rank band of the stated
bound (tests/archive_pool_ref.py), and newsrec_b200.pool_eval end to end for both families."""
import os

import numpy as np
import pytest
import torch

import archive_pool_ref as AR
import test_gpu_evaluate as TE
from test_gpu_predict import _model
from test_gpu_recommend_archive import SHAPES, _csr, _users

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def _lists(A, C_, dnn, excl):
    from newsrec_b200.ops import top_k_scores
    rows, offs = _csr(excl)
    return top_k_scores(_users(A), C_, C_.shape[0], rows, offs, dnn=dnn)


@pytest.mark.parametrize("P,F,hid", SHAPES)
def test_single_and_many_targets_equal_the_list_positions(P, F, hid):
    from newsrec_b200.ops import pool_ranks
    U, n = 40, 110
    g = torch.Generator().manual_seed(P * 7 + F)
    A, C_, dnn = AR.operands(g, U, P, F, hid, n)
    rng = np.random.default_rng(P + F)
    excl = [rng.choice(n, size=int(rng.integers(0, 6)), replace=False).tolist() for _ in range(U)]
    idx, score = _lists(A, C_, dnn, excl)
    idx, score = idx.cpu().numpy(), score.cpu().numpy()
    # one target per query: its rank is its position in nr_topk_archive's list over the pool without the exclusions
    tgt = [int(idx[u, rng.integers(0, n - len(excl[u]))]) for u in range(U)]
    xr, xo = _csr(excl)
    r, s = pool_ranks(_users(A), C_, torch.tensor(tgt), torch.arange(U + 1), xr, xo, dnn=dnn)
    for u in range(U):
        pos = int(np.flatnonzero(idx[u] == tgt[u])[0])
        assert int(r[u]) == pos and float(s[u]) == score[u, pos], (u, int(r[u]), pos)
    # 100 targets of one query (4 kernel rows) equal 100 single-target queries with the other 99 excluded
    u = 3
    many = rng.choice(n, size=100, replace=False)
    r100, s100 = pool_ranks(_users(A[u:u + 1]), C_, torch.from_numpy(many), torch.tensor([0, 100]), dnn=dnn)
    single_x = [[int(x) for x in many if x != t] for t in many]
    xr, xo = _csr(single_x)
    r1, s1 = pool_ranks(_users(A[u:u + 1].expand(100, -1, -1)), C_, torch.from_numpy(many), torch.arange(101), xr, xo, dnn=dnn)
    assert torch.equal(r100, r1) and torch.equal(s100, s1)


@pytest.mark.parametrize("P,F,hid", [(5, 300, 24), (1, 150, 17), (32, 400, 32)])
def test_ranks_lie_in_the_band_of_the_bound(P, F, hid):
    from newsrec_b200.ops import pool_ranks
    U, n = 2 * (64 // P) + 1, 5000
    g = torch.Generator().manual_seed(P + 99)
    A, C_, dnn = AR.operands(g, U, P, F, hid, n)
    rng = np.random.default_rng(P)
    counts = rng.integers(0, 40, size=U)
    tgt = [rng.choice(n, size=int(c), replace=False) for c in counts]
    rows = np.concatenate(tgt).astype(np.int64)
    offs = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    excl = [rng.choice(n, size=int(rng.integers(0, 30)), replace=False).tolist() for _ in range(U)]
    xr, xo = _csr(excl)
    rank, score = pool_ranks(_users(A), C_, torch.from_numpy(rows), torch.from_numpy(offs), xr, xo, dnn=dnn)
    again = pool_ranks(_users(A), C_, torch.from_numpy(rows), torch.from_numpy(offs), xr, xo, dnn=dnn)
    assert torch.equal(rank, again[0]) and torch.equal(score, again[1])
    S, E = AR.exact_and_bound(A, C_, dnn, DEV)
    S, E, rank, score = S.cpu().numpy(), E.cpu().numpy(), rank.cpu().numpy(), score.cpu().numpy()
    for q in range(U):
        elig = np.ones(n, bool)
        elig[excl[q]] = False
        elig[tgt[q]] = False
        for j, t in enumerate(tgt[q]):
            i = offs[q] + j
            assert abs(float(score[i]) - S[q, t]) <= E[q, t]
            lo = int(((S[q] - S[q, t] > E[q] + E[q, t]) & elig).sum())
            hi = int(((S[q] - S[q, t] >= -(E[q] + E[q, t])) & elig).sum())
            assert lo <= rank[i] <= hi, (q, t, lo, int(rank[i]), hi)


def test_flags_raise():
    from newsrec_b200.ops import pool_ranks
    g = torch.Generator().manual_seed(8)
    A, C_, dnn = AR.operands(g, 6, 5, 300, 24, 300)
    with pytest.raises(IndexError):
        pool_ranks(A, C_, torch.tensor([1, 300]), torch.tensor([0, 1, 2, 2, 2, 2, 2]), dnn=dnn)
    with pytest.raises(IndexError):
        xr, xo = _csr([[5], [], [-1], [], [], []])
        pool_ranks(A, C_, torch.tensor([1, 4]), torch.tensor([0, 1, 1, 2, 2, 2, 2]), xr, xo, dnn=dnn)
    bad = A.clone()
    bad[0, 1, 3] = float("nan")
    with pytest.raises(ValueError, match="not finite"):
        pool_ranks(bad, C_, torch.tensor([4]), torch.tensor([0, 1, 1, 1, 1, 1, 1]), dnn=dnn)


def test_raw_target_flag():
    import ctypes as C
    import newsrec_b200
    lib = newsrec_b200.load_library()
    g = torch.Generator().manual_seed(9)
    A, C_, dnn = AR.operands(g, 2, 3, 52, 11, 100)
    A, C_ = A.to(DEV).contiguous(), C_.to(DEV).contiguous()
    W1, b1, w2, b2 = (t.to(DEV).float().contiguous() for t in dnn)
    to = torch.tensor([0, 33, 34], dtype=torch.int64, device=DEV)
    tr = torch.arange(34, dtype=torch.int64, device=DEV)
    rank = torch.zeros(34, dtype=torch.int64, device=DEV)
    score = torch.zeros(34, dtype=torch.float32, device=DEV)
    flags = torch.zeros(3, dtype=torch.int32, device=DEV)
    nb = lib.nr_pool_ranks_archive_workspace(2, 3, 100, 52, 11)
    ws = torch.zeros(nb, dtype=torch.uint8, device=DEV)
    P_ = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    assert lib.nr_pool_ranks_archive(P_(A), 2, 3, P_(C_), 100, 52, P_(W1), P_(b1), 11, P_(w2), P_(b2), P_(to), P_(tr), None, None,
                                     P_(rank), P_(score), P_(flags[0:1]), P_(flags[1:2]), P_(flags[2:3]), P_(ws), nb,
                                     C.c_void_p(torch.cuda.current_stream().cuda_stream)) == 0
    torch.cuda.synchronize()
    assert flags.tolist() == [0, 0, 1]
    assert (rank[:33] == -1).all() and 0 <= int(rank[33]) < 100


@pytest.mark.parametrize("name", ["HiFiArk", "DKN"])
def test_evaluate_pool_matches_a_host_recompute_and_recommend(name, tmp_path):
    from newsrec_b200 import evaluate as E
    from newsrec_b200.pool_eval import evaluate_pool, metrics, pool_positions, positions
    from newsrec_b200.recommend import recommend
    d = str(tmp_path)
    TE._write_validation_dir(d)
    u2i = os.path.join(d, "user2int.tsv")
    model = _model(name)
    out = evaluate_pool(model, d, (1, 5, 10, 50), user2int_path=u2i)
    assert out == evaluate_pool(model, d, (1, 5, 10, 50), user2int_path=u2i, chunk_impressions=3)
    imp, rows, offsets, rank, score = pool_positions(model, d, user2int_path=u2i)
    with torch.no_grad():
        index, matrix = E.news_matrix(model, d)
        t = E.build_tables(d, index, model.config.num_clicked_news_a_user, 10 ** 9, u2i)
        pad = index["PADDED_NEWS"]
        from newsrec_b200.recommend import _Users, pool_operands
        users, dnn = pool_operands(model, _Users(t.user, t.history, t.history_length), matrix, E.new_flag(matrix.device))
        A = users if users.dim() == 3 else users.unsqueeze(1)
        S, Eb = AR.exact_and_bound(A, matrix[:pad], dnn, DEV)
        S, Eb = S.cpu().numpy(), Eb.cpu().numpy()
    for i, s in enumerate(imp):
        u = t.seg_user[s]
        pos = rows[offsets[i]:offsets[i + 1]]
        elig = np.ones(pad, bool)
        elig[[r for r in t.history[u] if r != pad]] = False
        elig[pos] = False
        for j, p in enumerate(pos):
            e = 2 * (Eb[u] + Eb[u, p]) + 1e-6 * abs(S[u, p])
            lo = int(((S[u] - S[u, p] > e) & elig).sum())
            hi = int(((S[u] - S[u, p] >= -e) & elig).sum())
            assert lo <= rank[offsets[i] + j] <= hi
    assert out == metrics(positions(rank, score, rows, offsets), offsets, (1, 5, 10, 50))
    # recommend's lists agree with the ranks: a positive with position c < k that is not in the user's history sits at
    # place c of the user's list over the pool when no other positive of its impression comes before it
    recs = str(tmp_path / "rec.tsv")
    recommend(model, d, recs, 50, user2int_path=u2i)
    ids = E.read_news(d, [])[0]
    lines = [[ids.index(x) for x in ln.split("\t")[1].split(",")] for ln in open(recs).read().splitlines()]
    beh = E.read_behaviors(d)
    hist_rows = {hs: r for r, hs in enumerate(E.distinct_histories(beh)["clicked_news"].tolist())}
    checked = 0
    for i, s in enumerate(imp):
        u = hist_rows[beh["clicked_news"].iloc[s]]
        lst, pos = lines[u], rows[offsets[i]:offsets[i + 1]]
        for j, p in enumerate(pos):
            c = int(rank[offsets[i] + j])
            if p in t.history[u] or c + len(pos) >= 50:
                continue
            # the list holds the other positives too: p's place is its rank plus the positives listed before it
            assert p in lst, (i, p, c)
            assert lst.index(p) == c + sum(1 for q in pos if q in lst[:lst.index(p)])
            checked += 1
    assert checked > 0
