"""Ranks over the whole pool on the H100: nr_pool_ranks / ops.pool_ranks against the band include/newsrec_b200.h states (an
fp64 brute force on the same fp32 inputs), against nr_topk_dot's own order, and newsrec_b200.pool_eval end to end.

Band: with e(n) = (2^-15 + 3 round_up(D, 64) 2^-23) sum_i |q_i||n_i| and S the fp64 product,
    |{n eligible : S(n) - S(t) > e(n) + e(t)}|  <=  rank(q, t)  <=  |{n eligible : S(n) - S(t) >= -(e(n) + e(t))}|
where the eligible news of q are the pool without its exclusions and its targets."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import gpu_checks as G
import test_gpu_evaluate as TE

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def _coeff(D):
    return 2.0 ** -15 + 3 * ((D + 63) // 64 * 64) * 2.0 ** -23


def _csr(lists):
    offs = np.zeros(len(lists) + 1, np.int64)
    offs[1:] = np.cumsum([len(x) for x in lists])
    rows = np.concatenate([np.asarray(x, np.int64) for x in lists]) if offs[-1] else np.zeros(0, np.int64)
    return torch.from_numpy(rows), torch.from_numpy(offs)


def _ranks(users, news, targets, excl=None):
    from newsrec_b200.ops import pool_ranks
    tr, to = _csr(targets)
    xr, xo = _csr(excl) if excl is not None else (None, None)
    r, s = pool_ranks(users, news, tr, to, xr, xo)
    return r.cpu().numpy(), s.cpu().numpy()


def _check_band(users, news, targets, excl=None):
    """ops.pool_ranks, every rank inside the band and every score within e(t) of S(t); returns (rank, score)."""
    rank, score = _ranks(users, news, targets, excl)
    D = users.shape[1]
    u64, n64 = users.double().to(DEV), news.double().to(DEV)
    i = 0
    for q, tq in enumerate(targets):
        if not len(tq):
            continue
        S = n64 @ u64[q]
        E = _coeff(D) * (n64.abs() @ u64[q].abs())
        elig = torch.ones(len(news), dtype=torch.bool, device=DEV)
        elig[torch.as_tensor(np.asarray(tq, np.int64), device=DEV)] = False
        if excl is not None and len(excl[q]):
            elig[torch.as_tensor(np.asarray(excl[q], np.int64), device=DEV)] = False
        for t in tq:
            d, e = S - S[t], E + E[t]
            lo, hi = int((elig & (d > e)).sum()), int((elig & (d >= -e)).sum())
            assert lo <= rank[i] <= hi, (q, t, lo, int(rank[i]), hi)
            assert abs(float(score[i]) - float(S[t])) <= float(E[t]), (q, t)
            i += 1
    assert i == len(rank)
    return rank, score


def _data(Q, n, D, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(Q, D, generator=g), torch.randn(n, D, generator=g)


@pytest.mark.parametrize("Q,n,D", [(1, 1, 300), (63, 127, 300), (65, 129, 150), (130, 97, 64), (200, 5000, 300),
                                   (3, 20_000, 300), (9000, 300, 100)])
def test_ranks_inside_the_band(Q, n, D):
    users, news = _data(Q, n, D, Q + n + D)
    rng = np.random.default_rng(Q + n)
    targets = [rng.choice(n, min(n, int(rng.integers(0, 4))), replace=False) for _ in range(Q)]
    excl = [rng.integers(0, n, int(rng.integers(0, 60))) for _ in range(Q)]
    for q in range(0, Q, 97):  # rows 0, 63, 64 and n - 1 among the targets
        targets[q] = np.unique(np.array([0, min(63, n - 1), min(64, n - 1), n - 1]))
    if Q > 2000:  # the band brute force on a sample of the rows; the kernel runs all of them
        keep = set(range(0, Q, 37))
        targets = [t if q in keep else np.zeros(0, np.int64) for q, t in enumerate(targets)]
    _check_band(users, news, targets, excl)
    _check_band(users, news, targets)


def test_single_targets_agree_with_top_k_exactly():
    from newsrec_b200.ops import top_k_scores
    for Q, n, D in ((70, 400, 300), (5, 30_000, 150)):  # one split, several
        users, news = _data(Q, n, D, 11 + Q)
        S = users.double() @ news.double().T
        rng = np.random.default_rng(Q)
        targets, excl = [], []
        for q in range(Q):
            order = torch.argsort(S[q], descending=True).numpy()
            t = int(order[int(rng.integers(0, 200))])      # mostly within the top 128
            targets.append([t])
            x = rng.choice(order[:300], 30, replace=False)
            excl.append(x[x != t])
        rank, score = _ranks(users, news, targets, excl)
        xr, xo = _csr(excl)
        idx, sc = top_k_scores(users, news, 128, xr, xo)
        idx, sc = idx.cpu().numpy(), sc.cpu().numpy()
        listed = 0
        for q in range(Q):
            hit = np.flatnonzero(idx[q] == targets[q][0])
            if len(hit):
                assert rank[q] == hit[0] and score[q] == sc[q, hit[0]], (q, rank[q], hit)
                listed += 1
            else:
                assert rank[q] >= 128, (q, rank[q])
        assert listed >= Q // 2


def test_duplicates_edges_excluded_targets_and_exclusion_forms():
    Q, n, D = 66, 4097, 300
    users, news = _data(Q, n, D, 21)
    t0 = 1000
    for r in (5, 999, 1001, 4096):  # identical copies of the target: equal scores, ordered by row
        news[r] = news[t0]
    targets = [[t0]] * Q
    _check_band(users, news, targets)
    # the target excluded as well: the same rank
    r2, s2 = _ranks(users, news, targets, [[t0, 7]] * Q)
    r3, s3 = _ranks(users, news, targets, [[7]] * Q)
    assert np.array_equal(r2, r3) and np.array_equal(s2.view(np.int32), s3.view(np.int32))
    # unsorted, duplicated and empty exclusions give the sorted set's ranks
    rng = np.random.default_rng(3)
    raw = [rng.integers(0, n, 80) for _ in range(Q)]
    raw = [np.concatenate([x, x[:10]]) if q % 3 else (np.zeros(0, np.int64) if q % 2 else x) for q, x in enumerate(raw)]
    a = _ranks(users, news, targets, raw)
    b = _ranks(users, news, targets, [np.unique(x) for x in raw])
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1].view(np.int32), b[1].view(np.int32))
    # the copies and the edge rows as targets: exactly their place in top_k's list
    from newsrec_b200.ops import top_k_scores
    for t in (0, 63, 64, 999, t0, 1001, n - 1):
        r, _ = _ranks(users[:3], news, [[t]] * 3)
        idx, _ = top_k_scores(users[:3], news, 128)
        for q in range(3):
            hit = np.flatnonzero(idx[q].cpu().numpy() == t)
            assert (len(hit) and r[q] == hit[0]) or (not len(hit) and r[q] >= 128), (t, q, r[q], hit)


def test_a_query_of_100_targets_equals_100_single_target_queries_and_runs_are_identical():
    Q, n, D = 4, 9000, 300
    users, news = _data(Q, n, D, 31)
    rng = np.random.default_rng(31)
    targets = [rng.choice(n, 100, replace=False) for _ in range(Q)]
    excl = [rng.integers(0, n, 40) for _ in range(Q)]
    rank, score = _check_band(users, news, targets, excl)
    rows = np.repeat(np.arange(Q), 100)
    single_t = [[t] for tq in targets for t in tq]
    single_x = [np.concatenate([excl[q], np.setdiff1d(targets[q], [t])]) for q, tq in enumerate(targets) for t in tq]
    r1, s1 = _ranks(users[torch.from_numpy(rows)], news, single_t, single_x)
    assert np.array_equal(rank, r1) and np.array_equal(score.view(np.int32), s1.view(np.int32))
    again = _ranks(users, news, targets, excl)
    assert np.array_equal(rank, again[0]) and np.array_equal(score.view(np.int32), again[1].view(np.int32))


def test_flags_raise():
    from newsrec_b200.ops import pool_ranks
    users, news = _data(3, 500, 100, 41)
    tr, to = _csr([[1], [2, 3], []])
    with pytest.raises(IndexError, match="outside the news pool"):
        pool_ranks(users, news, torch.tensor([1, 500, 3]), to)
    with pytest.raises(IndexError, match="outside the news pool"):
        pool_ranks(users, news, tr, to, *_csr([[4], [-1], []]))
    bad = news.clone()
    bad[77, 3] = float("nan")
    with pytest.raises(ValueError, match="not finite"):
        pool_ranks(users, bad, tr, to)


def test_raw_entry_point_guards_limits_and_refusals():
    from newsrec_b200 import NewsrecError, launch_count, load_library
    from newsrec_b200.ops import pool_ranks
    lib = load_library()
    Q, n, D = 70, 3000, 150
    users, news = (x.to(DEV) for x in _data(Q, n, D, 51))
    lists = [[q % n, (7 * q + 1) % n] for q in range(Q)]
    lists[5] = list(range(33))                                     # more than 32 targets: rank -1, target flag
    tr, to = (x.to(DEV) for x in _csr(lists))
    T = len(tr)
    ws_bytes = int(lib.nr_pool_ranks_workspace(Q, n, D))
    assert ws_bytes > 0 and lib.nr_pool_ranks_workspace(Q, 0, D) == -1 and lib.nr_pool_ranks_workspace(Q, n, 4097) == -1
    rank = G._Guarded(T, torch.int64, -777, sentinel=-4242)
    score = G._Guarded(T, torch.float32, float("nan"))
    ws = G._Guarded(ws_bytes + 256, torch.uint8, 0xAB, sentinel=0x5C)
    flags = G._Guarded(3, torch.int32, 0, sentinel=-3)
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    wp = ws.all.data_ptr()
    pad = (-wp) % 256
    fp = flags.all.data_ptr()

    def call(ld=D, d=D, nn=n, wsb=ws_bytes):
        return lib.nr_pool_ranks(users.data_ptr(), Q, ld, news.data_ptr(), nn, D, d, to.data_ptr(), tr.data_ptr(), None, None,
                                 rank.all.data_ptr(), score.all.data_ptr(), fp, fp + 4, fp + 8, wp + pad, wsb, s)

    assert call() == 0
    torch.cuda.synchronize()
    assert rank.guard_ok() and score.guard_ok() and flags.guard_ok() and ws.guard_ok()
    assert flags.body.tolist() == [0, 0, 1]
    r = rank.body.cpu().numpy()
    a, b = int(to[5]), int(to[6])
    assert (r[a:b] == -1).all() and (np.delete(r, np.arange(a, b)) >= 0).all()
    ok = [lst if q != 5 else [] for q, lst in enumerate(lists)]
    want, want_s = _ranks(users, news, ok)
    assert np.array_equal(np.delete(r, np.arange(a, b)), want)
    assert np.array_equal(np.delete(score.body.cpu().numpy(), np.arange(a, b)).view(np.int32), want_s.view(np.int32))
    n0 = launch_count()
    for bad in [dict(d=0), dict(d=4097), dict(ld=D - 1), dict(nn=0), dict(wsb=ws_bytes - 1)]:
        before = (rank.body.clone(), score.body.clone())
        assert call(**bad) == -1 and lib.nr_last_error().decode().startswith("nr_pool_ranks"), bad
        torch.cuda.synchronize()
        assert torch.equal(rank.body, before[0]) and G._bits_equal(score.body, before[1])
    assert lib.nr_pool_ranks(users.data_ptr(), Q, D, news.data_ptr(), n, D, D, None, tr.data_ptr(), None, None,
                             rank.all.data_ptr(), score.all.data_ptr(), fp, fp + 4, fp + 8, wp + pad, ws_bytes, s) == -1
    with pytest.raises(NewsrecError):
        pool_ranks(users, news[:, :10], tr, to)
    with pytest.raises(NewsrecError):
        pool_ranks(users, news, tr, to[:-1])
    assert launch_count() == n0
    assert rank.guard_ok() and score.guard_ok() and ws.guard_ok()


# ------------------------------------------------------------------------------------------------------------------------
# end to end
# ------------------------------------------------------------------------------------------------------------------------
FAMILIES = {"NRMS": "nrms", "LSTUR": "lstur_ini", "NAML": "naml"}


def _model(name):
    torch.manual_seed(0)
    model, cfg = G.build_model(FAMILIES[name], V=TE.V, ncat=TE.NCAT, nusers=TE.NUSERS, H=TE.H)
    cfg.batch_size = 2
    return model.eval()


@pytest.mark.parametrize("name", list(FAMILIES))
def test_evaluate_pool_chunks_host_recompute_and_recommend(name, tmp_path):
    from newsrec_b200 import evaluate as E
    from newsrec_b200 import pool_eval as P
    from newsrec_b200.recommend import recommend
    d = str(tmp_path)
    TE._write_validation_dir(d)
    u2i = os.path.join(d, "user2int.tsv")
    model = _model(name)
    ks = (1, 5, 20, 100, 1000)
    res = {c: P.evaluate_pool(model, d, ks, user2int_path=u2i, chunk_impressions=c) for c in (1, 7, 10 ** 9)}
    assert res[1] == res[7] == res[10 ** 9], res
    m = res[1]
    assert m["impressions"] > 30 and m["recall@1000"] == 1.0 and 0 < m["mrr"] <= 1
    imp, rows, offsets, rank, score = P.pool_positions(model, d, user2int_path=u2i, chunk_impressions=7)
    c = P.positions(rank, score, rows, offsets)
    assert P.metrics(c, offsets, ks) == m
    # host recompute from fp64 scores wherever no eligible news lies within the band
    with torch.no_grad():
        index, matrix = E.news_matrix(model, d)
        t = E.build_tables(d, index, model.config.num_clicked_news_a_user, 10 ** 9, u2i)
        uv = E.user_vectors(model, t, matrix, E.new_flag(matrix.device))
    pad = index["PADDED_NEWS"]
    pool = matrix[:pad].double()
    checked = 0
    for s_ in range(len(imp)):
        u = int(t.seg_user[imp[s_]])
        S = (pool @ uv[u].double()).cpu().numpy()
        Eb = (_coeff(pool.shape[1]) * (pool.abs() @ uv[u].double().abs())).cpu().numpy()
        P_i = rows[offsets[s_]:offsets[s_ + 1]]
        hist = set(int(r) for r in t.history[u] if r != pad)
        elig = np.array([r not in hist and r not in set(P_i.tolist()) for r in range(pad)])
        for j, p in enumerate(P_i):
            near = elig & (np.abs(S - S[p]) <= Eb + Eb[p])
            others = np.array([q for q in P_i if q != p], np.int64)
            if near.any() or (np.abs(S[others] - S[p]) <= Eb[others] + Eb[p]).any():
                continue
            host = int((elig & (S > S[p])).sum()) + int((S[others] > S[p]).sum())
            assert c[offsets[s_] + j] == host, (s_, p, c[offsets[s_] + j], host)
            checked += 1
    assert checked >= 40
    # recommend's list: a positive in a user's top-k line has c_p < k
    k = 20
    out = str(tmp_path / "rec.tsv")
    recommend(model, d, out, k, user2int_path=u2i)
    lines = [ln.split("\t")[1] for ln in open(out).read().splitlines()]
    ids = E.read_news(d, [])[0]
    listed = 0
    for s_ in range(len(imp)):
        top = lines[int(t.seg_user[imp[s_]])].split(",")
        for j, p in enumerate(rows[offsets[s_]:offsets[s_ + 1]]):
            if ids[p] in top:
                assert c[offsets[s_] + j] < k
                listed += 1
    assert listed > 0
    # the clicked news kept in the pool: every rank at least as large
    kept = P.pool_positions(model, d, exclude_clicked=False, user2int_path=u2i)
    assert (kept[3] >= rank).all()
