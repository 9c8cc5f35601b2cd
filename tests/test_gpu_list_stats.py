"""nr_list_stats / ops.list_stats and newsrec_b200.pool_eval.evaluate_lists on the H100.

The kernel against fp64 on the same fp32 rows: every pair sum within the header's bound (pairs x e_sim, e_sim nr_mmr_rerank's
similarity bound), distinct counts exact, two runs bit-identical, refusals before any launch with the outputs untouched.
evaluate_lists end to end: plain lists kept with the clicked news give evaluate_pool's recall@K and nDCG@K exactly (both
orders come from the same score bits) and the MRR of pool_positions truncated at k; capped lists against the plain
restatement of tests/list_eval_ref.py on the lists top_k_scores returns; MMR at lambda = 1 is the plain result; the result
does not depend on chunk_impressions, bit for bit."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import gpu_checks as G
import list_eval_ref as R
import mmr_ref as M
import test_gpu_evaluate as TE
import test_gpu_recommend as TR
from test_gpu_predict import _model as _predict_model

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def _news(n, D, seed, zero=(0, 1)):
    news = torch.randn(n, D, generator=torch.Generator().manual_seed(seed))
    news[list(zero)] = 0.0
    return news.to(DEV)


def _lists(R_, k, n, seed):
    """Rows of k entries with -1 tails at every length 0 .. k (garbage after the first -1), repeated rows and zero rows."""
    g = np.random.default_rng(seed)
    lists = g.integers(0, n, (R_, k))
    for r in range(R_):
        L = r % (k + 1)
        if L < k:
            lists[r, L] = -1
            lists[r, L + 1:] = g.choice([-1, -7, n, n + 3, 5], k - L - 1)   # ignored
        if r % 3 == 0 and L >= 3:
            lists[r, 2] = lists[r, 0]                                      # a repeated row
        if r % 4 == 1 and L >= 2:
            lists[r, 1] = 0                                                # an all-zero row
    return torch.from_numpy(lists).to(DEV)


def _exact(news, lists, ks, cats=None):
    """(pair_sum fp64 of exact cosines, distinct, pairs) per row and cut-off."""
    X = news.double()
    nrm = X.norm(dim=1, keepdim=True)
    Xn = torch.where(nrm > 0, X / nrm.clamp_min(1e-300), torch.zeros_like(X))
    li = lists.cpu().numpy()
    ps = np.zeros((len(li), len(ks)))
    dc = np.zeros((len(li), len(ks)), np.int64)
    pairs = np.zeros((len(li), len(ks)))
    for r, row in enumerate(li):
        live = R.live(row)
        if len(live) >= 2:
            sub = Xn[torch.tensor(live, device=DEV)]
            Cm = torch.tril(sub @ sub.T, diagonal=-1)
            pref = Cm.sum(1).cumsum(0).cpu().numpy()
        for c, K in enumerate(ks):
            Kp = min(K, len(live))
            ps[r, c] = pref[Kp - 1] if Kp >= 2 else 0.0
            pairs[r, c] = Kp * (Kp - 1) / 2
            if cats is not None:
                dc[r, c] = len({int(cats[x]) for x in live[:Kp]})
    return ps, dc, pairs


def _ks_sets(k):
    g = np.random.default_rng(k)
    sets = [(k,), tuple(sorted({1, k}))]
    if k > 8:
        sets.append(tuple(sorted(set(g.choice(np.arange(1, k), 7, replace=False).tolist()) | {k})))
        sets.append(tuple(sorted(g.choice(np.arange(1, k + 1), 8, replace=False).tolist())))
    return sets


@pytest.mark.parametrize("D", [1, 63, 300, 4096])
@pytest.mark.parametrize("k", [1, 2, 37, 64, 65, 128])
def test_kernel_against_fp64(k, D):
    from newsrec_b200.ops import list_stats
    n = 400
    news = _news(n, D, seed=k * 7 + D)
    lists = _lists(2 * (k + 1) + 5, k, n, seed=k + D)
    cats = torch.from_numpy(np.random.default_rng(D).integers(-6, 5, n).astype(np.int32))
    cats[:50] = -2 ** 31 + torch.arange(50, dtype=torch.int32) % 3         # extreme negative keys
    e = M.e_sim(D)
    for ks in _ks_sets(k):
        for cat in (None, cats):
            ps, dc = list_stats(news, lists, ks, categories=cat)
            ps2, dc2 = list_stats(news, lists, ks, categories=cat)
            assert torch.equal(ps.view(torch.int64), ps2.view(torch.int64))
            assert (dc is None) == (cat is None) and (dc is None or torch.equal(dc, dc2))
            want, want_d, pairs = _exact(news, lists, ks, None if cat is None else cat.numpy())
            err = np.abs(ps.cpu().numpy() - want)
            assert (err <= pairs * e + pairs ** 2 * 2.0 ** -52 + 1e-300).all(), (ks, err.max(), (err / np.maximum(pairs, 1)).max(), e)
            assert (ps.cpu().numpy()[pairs == 0] == 0).all()
            if cat is not None:
                assert np.array_equal(dc.cpu().numpy(), want_d), ks


def test_repeated_rows_are_cosine_one_and_zero_rows_zero():
    from newsrec_b200.ops import list_stats
    news = _news(20, 300, seed=1, zero=(3,))
    lists = torch.tensor([[5, 5, 5, -1], [3, 5, 3, 7], [9, 9, 9, 9]], device=DEV)
    ps, _ = list_stats(news, lists, (2, 3, 4))
    ps = ps.cpu().numpy()
    e = M.e_sim(300)
    assert abs(ps[0, 0] - 1) <= e and abs(ps[0, 1] - 3) <= 3 * e and ps[0, 2] == ps[0, 1]
    assert ps[1, 0] == 0 and ps[1, 1] == 0                                 # every pair holds the zero row
    assert abs(ps[2, 2] - 6) <= 6 * e


def test_refusals_leave_the_outputs_untouched_and_flags():
    from newsrec_b200 import NewsrecError, launch_count, load_library
    from newsrec_b200.ops import _p, _stream, list_stats
    lib = load_library()
    n, D, k, Rr = 50, 16, 6, 9
    news = _news(n, D, seed=2)
    lists = _lists(Rr, k, n, seed=3)
    cats = torch.arange(n, dtype=torch.int32, device=DEV) % 4
    ps = G._Guarded(Rr * 8, torch.float64, float("nan"))
    dc = G._Guarded(Rr * 8, torch.int32, -9, sentinel=-4242)
    flag = G._Guarded(1, torch.int32, 0, sentinel=-3)

    def ps_guard_ok():  # an fp64 buffer: compare its guard's bits as int64
        return torch.equal(ps.all[ps.n:].view(torch.int64), ps.guard.view(torch.int64))

    def call(ks=(2, 6), nn=n, d=D, ld=D, kk=k, rows=Rr, cat=True, dist=True, news_p=None, n_ks=None):
        arr = (C.c_int * max(len(ks), 1))(*ks)
        return lib.nr_list_stats(news.data_ptr() if news_p is None else news_p, nn, ld, d, lists.data_ptr(), rows, kk,
                                 cats.data_ptr() if cat else None, arr, len(ks) if n_ks is None else n_ks, ps.all.data_ptr(),
                                 dc.all.data_ptr() if dist else None, flag.all.data_ptr(), _stream())

    assert call() == 0
    torch.cuda.synchronize()
    assert ps_guard_ok() and dc.guard_ok() and flag.guard_ok() and int(flag.body[0]) == 0
    n0 = launch_count()
    for bad in [dict(d=0), dict(d=4097, ld=4097), dict(ld=D - 1), dict(kk=0), dict(kk=129), dict(ks=()), dict(ks=(1, 2), n_ks=9),
                dict(ks=tuple(range(1, 10)), kk=20), dict(ks=(3, 2)), dict(ks=(2, 2)), dict(ks=(0, 2)), dict(ks=(2, 7)),
                dict(rows=-1), dict(rows=2 ** 31 - 64), dict(nn=-1), dict(nn=2 ** 31 - 64), dict(cat=False), dict(dist=False),
                dict(news_p=0)]:
        before = (ps.body.clone(), dc.body.clone())
        assert call(**bad) == -1 and lib.nr_last_error().decode().startswith("nr_list_stats"), bad
        torch.cuda.synchronize()
        assert torch.equal(ps.body.view(torch.int64), before[0].view(torch.int64)) and torch.equal(dc.body, before[1]), bad
    assert call(rows=0) == 0                                               # nothing to do: no launch
    assert launch_count() == n0
    assert ps_guard_ok() and dc.guard_ok() and flag.guard_ok()
    for ks in ((), (0,), (3, 2), (1, 7), tuple(range(1, 10)), (1.5,)):
        with pytest.raises(NewsrecError):
            list_stats(news, lists, ks)
    with pytest.raises(NewsrecError):
        list_stats(news, lists, (2,), categories=torch.zeros(n - 1, dtype=torch.int32))
    # a live row outside the pool sets the flag; one after the first -1 does not
    for row, want in (([0, 1, n, 3, 4, 5], 1), ([0, -5, 2, 3, 4, 5], 1), ([0, 1, -1, n + 9, -7, 5], 0)):
        bad = torch.tensor([row, [1, 2, 3, 4, 5, 6]], device=DEV)
        if want:
            with pytest.raises(IndexError):
                list_stats(news, bad, (6,))
        else:
            list_stats(news, bad, (6,))


def _same(a, b):
    """Two result dicts with the same keys and the same bits (NaN included)."""
    assert set(a) == set(b), sorted(set(a) ^ set(b))
    for key in a:
        assert np.asarray(a[key], np.float64).view(np.int64) == np.asarray(b[key], np.float64).view(np.int64), (key, a[key], b[key])


def _split(tmp_path):
    d = str(tmp_path)
    TE._write_validation_dir(d)
    return d, os.path.join(d, "user2int.tsv")


@pytest.mark.parametrize("name", ["NRMS", "HiFiArk", "DKN"])
def test_plain_lists_agree_with_evaluate_pool(name, tmp_path):
    from newsrec_b200 import pool_eval as P
    d, u2i = _split(tmp_path)
    model = TR._model(name) if name == "NRMS" else _predict_model(name)
    k, ks = 20, (1, 5, 10, 20)
    got = P.evaluate_lists(model, d, k, ks, exclude_clicked=False, user2int_path=u2i)
    want = P.evaluate_pool(model, d, ks, exclude_clicked=False, user2int_path=u2i)
    assert got["impressions"] == want["impressions"] > 30
    for K in ks:
        assert got[f"recall@{K}"] == want[f"recall@{K}"] and got[f"ndcg@{K}"] == want[f"ndcg@{K}"], K
    imp, rows, offsets, rank, score = P.pool_positions(model, d, exclude_clicked=False, user2int_path=u2i)
    c = P.positions(rank, score, rows, offsets)
    first = np.full(len(imp), np.iinfo(np.int64).max)
    np.minimum.at(first, np.repeat(np.arange(len(imp)), np.diff(offsets)), c)
    assert got[f"mrr@{k}"] == np.float64(np.mean(np.where(first < k, 1.0 / (1.0 + first), 0.0)))
    assert got[f"recall@{k}"] > 0 and 0 < got[f"coverage@{k}"] <= 1 and 0 <= got[f"gini@{k}"] < 1
    assert got[f"list_length@{k}"] == k and 1 <= got[f"distinct_category@{k}"] <= k
    # a chunk of one impression and of seven: the same bits
    for chunk in (1, 7):
        _same(P.evaluate_lists(model, d, k, ks, exclude_clicked=False, user2int_path=u2i, chunk_impressions=chunk), got)


def _lists_of(model, d, u2i, k, **opts):
    """The lists top_k_scores returns for every counted impression (as evaluate_lists builds them, with the clicked news
    excluded), its positives, the pool and the category keys."""
    from newsrec_b200 import evaluate as E
    from newsrec_b200 import pool_eval as P
    from newsrec_b200.ops import top_k_scores
    from newsrec_b200.recommend import _Users, exclusion_csr, pool_operands
    with torch.no_grad():
        index, matrix = E.news_matrix(model, d)
        pad = index["PADDED_NEWS"]
        t = E.build_tables(d, index, model.config.num_clicked_news_a_user, 10 ** 9, u2i)
        users, dnn = pool_operands(model, _Users(t.user, t.history, t.history_length), matrix, E.new_flag(DEV))
    xr, xo = exclusion_csr(t.history, pad)
    idx, _ = top_k_scores(users, matrix[:pad], k, torch.from_numpy(xr), torch.from_numpy(xo), dnn=dnn, **opts)
    imp, rows, offsets = P.positives(t.cand, t.labels, t.seg_offsets)
    lists = idx.cpu().numpy()[t.seg_user[imp]]
    positives = [rows[offsets[i]:offsets[i + 1]].tolist() for i in range(len(imp))]
    return lists, positives, matrix[:pad], E.read_news(d, ["category"])[1]["category"]


@pytest.mark.parametrize("m", [1, 2])
def test_capped_lists_against_the_restatement(m, tmp_path):
    from newsrec_b200 import pool_eval as P
    d, u2i = _split(tmp_path)
    model = TR._model("NRMS")
    k, ks = 20, (1, 5, 20)
    got = P.evaluate_lists(model, d, k, ks, max_per_category=m, user2int_path=u2i)
    from newsrec_b200.evaluate import read_news
    cats = read_news(d, ["category"])[1]["category"]
    lists, positives, pool, _ = _lists_of(model, d, u2i, k, categories=torch.from_numpy(cats.astype(np.int32)).to(DEV),
                                          max_per_category=m)
    for row in lists:
        live = R.live(row)
        assert max(np.bincount(cats[live] - cats.min()), default=0) <= m
    if m == 1:                                                             # 11 categories: the caps shorten the lines
        assert max(len(R.live(r)) for r in lists) <= 11 < k
    ps, dc = R.list_stats(pool.cpu().numpy(), lists, ks, cats)
    want = R.metrics(lists, positives, pool.shape[0], ks, ps, dc)
    R.assert_close(got, want, tol={f"ils@{K}": M.e_sim(pool.shape[1]) for K in ks})
    assert got["distinct_category@20"] == want["distinct_category@20"]


def test_mmr_lambda_one_is_plain_and_chunks_do_not_matter(tmp_path):
    from newsrec_b200 import pool_eval as P
    d, u2i = _split(tmp_path)
    model = TR._model("NRMS")
    plain = P.evaluate_lists(model, d, 10, user2int_path=u2i)
    _same(P.evaluate_lists(model, d, 10, mmr_lambda=1.0, user2int_path=u2i), plain)
    mmr = {c: P.evaluate_lists(model, d, 10, mmr_lambda=0.5, mmr_depth=40, user2int_path=u2i, chunk_impressions=c)
           for c in (1, 7, P.DEFAULT_CHUNK)}
    _same(mmr[1], mmr[7])
    _same(mmr[1], mmr[P.DEFAULT_CHUNK])
    lists, positives, pool, cats = _lists_of(model, d, u2i, 10, mmr_lambda=0.5, mmr_depth=40)
    ps, dc = R.list_stats(pool.cpu().numpy(), lists, (5, 10), cats)
    R.assert_close(mmr[1], R.metrics(lists, positives, pool.shape[0], (5, 10), ps, dc),
                   tol={f"ils@{K}": M.e_sim(pool.shape[1]) for K in (5, 10)})


def test_mmr_lowers_intra_list_similarity_on_a_clustered_pool():
    from newsrec_b200.ops import list_stats, top_k_scores
    g = torch.Generator().manual_seed(5)
    stories = torch.randn(50, 64, generator=g)
    news = (stories[torch.randint(0, 50, (3000,), generator=g)] + 0.15 * torch.randn(3000, 64, generator=g)).to(DEV)
    users = torch.randn(500, 64, generator=g).to(DEV)
    ils = {}
    for lam in (1.0, 0.5):
        idx, _ = top_k_scores(users, news, 10, mmr_lambda=lam, mmr_depth=40)
        ps, _ = list_stats(news, idx, (10,))
        ils[lam] = float(ps.mean()) / 45
    assert ils[0.5] < ils[1.0], ils
