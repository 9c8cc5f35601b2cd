"""Time windows over the pool on the H100: the ranged top-k and rank kernels (nr_topk_dot_ranged, nr_topk_archive_ranged,
nr_pool_ranks_ranged, nr_pool_ranks_archive_ranged) bit for bit against the unranged calls with the complement of each
range excluded, bad ranges, and recommend / evaluate_pool / evaluate_lists with max_age_hours end to end against an fp64
restatement of the window's definition (newsrec_b200.window)."""
import os

import numpy as np
import pytest
import torch

import archive_pool_ref as AR
import test_gpu_evaluate as TE
from test_gpu_predict import _model

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def _csr(lists):
    offs = np.zeros(len(lists) + 1, np.int64)
    offs[1:] = np.cumsum([len(x) for x in lists])
    rows = np.concatenate([np.asarray(x, np.int64) for x in lists]) if offs[-1] else np.zeros(0, np.int64)
    return torch.from_numpy(rows), torch.from_numpy(offs)


def _ranges(U, n, k, rng):
    """Per-row [lo, hi): empty, the whole pool, one row, mid-tile and 64-row edges, shorter than k, then random ones."""
    fixed = [(0, 0), (n // 2, n // 2), (0, n), (5, 6), (n - 1, n), (30, 97), (64, 128), (0, 64), (64 * (n // 128), n),
             (100, 100 + max(1, k // 2)), (63, 65), (1, n - 1)]
    lo, hi = np.zeros(U, np.int64), np.zeros(U, np.int64)
    for u in range(U):
        if u < len(fixed):
            lo[u], hi[u] = fixed[u]
        else:
            a, b = sorted(rng.integers(0, n + 1, 2))
            lo[u], hi[u] = a, b
    return lo, hi


def _with_complement(excl, lo, hi, n):
    return [sorted(set(e) | set(range(0, int(a))) | set(range(int(b), n))) for e, a, b in zip(excl, lo, hi)]


def _excl(U, n, rng, on):
    return [rng.choice(n, size=int(rng.integers(0, 40)), replace=False).tolist() if on else [] for _ in range(U)]


def _same(a, b):
    assert torch.equal(a[0], b[0]), "idx"
    assert torch.equal(a[1].view(torch.int32), b[1].view(torch.int32)), "score bits"


def _users(A):
    return A[:, 0] if A.shape[1] == 1 else A


# U = 5: the planner splits the 16 news tiles; U = 9000 (dot) / 141 blocks (archive): one split
@pytest.mark.parametrize("U", [5, 9000])
@pytest.mark.parametrize("cap", [None, 2])
def test_top_k_dot_ranged_equals_the_complement_excluded(U, cap):
    from newsrec_b200.ops import top_k_scores
    n, D, k = 1000, 300, 10
    g = torch.Generator().manual_seed(U + (cap or 0))
    users, news = torch.randn(U, D, generator=g), torch.randn(n, D, generator=g)
    rng = np.random.default_rng(U)
    lo, hi = _ranges(U, n, k, rng)
    opts = {} if cap is None else dict(categories=torch.from_numpy(rng.integers(0, 7, n)), max_per_category=cap)
    for on in (False, True):
        excl = _excl(U, n, rng, on)
        got = top_k_scores(users, news, k, *_csr(excl), row_range=(torch.from_numpy(lo), torch.from_numpy(hi)), **opts)
        _same(got, top_k_scores(users, news, k, *_csr(_with_complement(excl, lo, hi, n)), **opts))
        whole = (torch.zeros(U, dtype=torch.int64), torch.full((U,), n, dtype=torch.int64))
        _same(top_k_scores(users, news, k, *_csr(excl), row_range=whole, **opts), top_k_scores(users, news, k, *_csr(excl), **opts))
    _same(top_k_scores(users, news, k, row_range=whole, **opts), top_k_scores(users, news, k, **opts))


@pytest.mark.parametrize("P,U", [(1, 5), (1, 64 * 140), (5, 5), (5, 12 * 140)])
@pytest.mark.parametrize("cap", [None, 2])
def test_top_k_archive_ranged_equals_the_complement_excluded(P, U, cap):
    from newsrec_b200.ops import top_k_scores
    n, F, hid, k = 1000, 100, 16, 10
    g = torch.Generator().manual_seed(P * 31 + U)
    A, C_, dnn = AR.operands(g, U, P, F, hid, n)
    rng = np.random.default_rng(P + U)
    lo, hi = _ranges(U, n, k, rng)
    opts = {} if cap is None else dict(categories=torch.from_numpy(rng.integers(0, 7, n)), max_per_category=cap)
    rr = (torch.from_numpy(lo), torch.from_numpy(hi))
    for on in (False, True):
        excl = _excl(U, n, rng, on)
        got = top_k_scores(_users(A), C_, k, *_csr(excl), dnn=dnn, row_range=rr, **opts)
        _same(got, top_k_scores(_users(A), C_, k, *_csr(_with_complement(excl, lo, hi, n)), dnn=dnn, **opts))
    whole = (torch.zeros(U, dtype=torch.int64), torch.full((U,), n, dtype=torch.int64))
    _same(top_k_scores(_users(A), C_, k, dnn=dnn, row_range=whole, **opts), top_k_scores(_users(A), C_, k, dnn=dnn, **opts))


def _targets(U, n, lo, hi, excl, rng):
    """Per row: targets inside and outside its range, and some that are also excluded."""
    out = []
    for u in range(U):
        t = set(rng.choice(n, size=int(rng.integers(0, 5)), replace=False).tolist())
        if hi[u] > lo[u]:
            t |= set(rng.integers(lo[u], hi[u], 3).tolist())
        if excl[u]:
            t.add(excl[u][0])
        out.append(sorted(t))
    return out


@pytest.mark.parametrize("U", [5, 9000])
@pytest.mark.parametrize("dnn_P", [None, 1, 5])
def test_pool_ranks_ranged_equal_the_complement_excluded(U, dnn_P):
    from newsrec_b200.ops import pool_ranks
    n, k = 1000, 10
    g = torch.Generator().manual_seed(U + (dnn_P or 0))
    rng = np.random.default_rng(U + 7)
    if dnn_P is None:
        users, news, dnn = torch.randn(U, 300, generator=g), torch.randn(n, 300, generator=g), None
    else:
        U = U if dnn_P == 1 or U < 64 else 12 * 140
        A, news, dnn = AR.operands(g, U, dnn_P, 100, 16, n)
        users = _users(A)
    lo, hi = _ranges(U, n, k, rng)
    rr = (torch.from_numpy(lo), torch.from_numpy(hi))
    for on in (False, True):
        excl = _excl(U, n, rng, on)
        tr, to = _csr(_targets(U, n, lo, hi, excl, rng))
        got = pool_ranks(users, news, tr, to, *_csr(excl), dnn=dnn, row_range=rr)
        want = pool_ranks(users, news, tr, to, *_csr(_with_complement(excl, lo, hi, n)), dnn=dnn)
        assert torch.equal(got[0], want[0]) and torch.equal(got[1].view(torch.int32), want[1].view(torch.int32))
    whole = (torch.zeros(U, dtype=torch.int64), torch.full((U,), n, dtype=torch.int64))
    assert all(torch.equal(a, b) for a, b in zip(pool_ranks(users, news, tr, to, dnn=dnn, row_range=whole),
                                                 pool_ranks(users, news, tr, to, dnn=dnn)))


def _p(t):
    return None if t is None else t.data_ptr()


def test_bad_ranges_set_the_flag_and_leave_the_other_rows_alone():
    from newsrec_b200 import load_library
    from newsrec_b200.ops import pool_ranks, top_k_scores
    lib = load_library()
    U, n, D, k = 70, 1000, 300, 10
    g = torch.Generator().manual_seed(11)
    users, news = torch.randn(U, D, generator=g).to(DEV), torch.randn(n, D, generator=g).to(DEV)
    lo = torch.full((U,), 100, dtype=torch.int64)
    hi = torch.full((U,), 900, dtype=torch.int64)
    clean = top_k_scores(users, news, k, row_range=(lo, hi))
    tr, to = _csr([[5, 500]] * U)
    clean_r = pool_ranks(users, news, tr, to, row_range=(lo, hi))
    ws = torch.empty(max(int(lib.nr_topk_dot_workspace(U, n, D, k)), int(lib.nr_pool_ranks_workspace(U, n, D))),
                     dtype=torch.uint8, device=DEV)
    stream = torch.cuda.current_stream().cuda_stream
    for bad_row, (a, b) in ((3, (-1, 10)), (40, (0, n + 1)), (69, (600, 599))):
        blo, bhi = lo.clone(), hi.clone()
        blo[bad_row], bhi[bad_row] = a, b
        blo, bhi = blo.to(DEV), bhi.to(DEV)
        idx = torch.empty((U, k), dtype=torch.int64, device=DEV)
        score = torch.empty((U, k), dtype=torch.float32, device=DEV)
        flags = torch.zeros(3, dtype=torch.int32, device=DEV)
        assert lib.nr_topk_dot_ranged(_p(users), U, D, _p(news), n, D, D, k, None, None, None, 0, _p(blo), _p(bhi), _p(idx),
                                      _p(score), _p(flags[0:1]), _p(flags[1:2]), _p(ws), ws.numel(), stream) == 0
        assert flags.tolist()[:2] == [1, 0], (a, b)
        assert (idx[bad_row] == -1).all() and (score[bad_row] == float("-inf")).all()
        keep = torch.arange(U, device=DEV) != bad_row
        assert torch.equal(idx[keep], clean[0][keep]) and torch.equal(score[keep], clean[1][keep])
        rank = torch.empty(2 * U, dtype=torch.int64, device=DEV)
        rscore = torch.empty(2 * U, dtype=torch.float32, device=DEV)
        flags.zero_()
        d_to, d_tr = to.to(DEV), tr.to(DEV)
        assert lib.nr_pool_ranks_ranged(_p(users), U, D, _p(news), n, D, D, _p(d_to), _p(d_tr), None, None, _p(blo), _p(bhi),
                                        _p(rank), _p(rscore), _p(flags[0:1]), _p(flags[1:2]), _p(flags[2:3]), _p(ws),
                                        ws.numel(), stream) == 0
        assert flags.tolist() == [1, 0, 0]
        bad = torch.zeros(2 * U, dtype=torch.bool, device=DEV)
        bad[2 * bad_row:2 * bad_row + 2] = True
        assert (rank[bad] == -1).all()
        assert torch.equal(rank[~bad], clean_r[0].to(DEV)[~bad]) and torch.equal(rscore[~bad], clean_r[1].to(DEV)[~bad])
    with pytest.raises(IndexError, match="row range"):
        top_k_scores(users, news, k, row_range=(lo - 200, hi))
    with pytest.raises(IndexError, match="row range"):
        pool_ranks(users, news, tr, to, row_range=(lo, hi + 200))


# ------------------------------------------------------------------------------------------------------------------------
# end to end
# ------------------------------------------------------------------------------------------------------------------------
HOUR = 3600


def _stamp(h):
    """MIND time of hour h (0 .. 47) after 11/14/2019 12:00:00 AM."""
    day, hh = 14 + h // 24, h % 24
    ampm, h12 = ("AM" if hh < 12 else "PM"), (hh % 12 or 12)
    return f"11/{day}/2019 {h12}:00:00 {ampm}"


def _write_timed_split(d, shown_first=False):
    """TE's validation split with each impression at a whole hour (so windows of whole hours hit first-shown times exactly
    at both ends) and some news never listed; shown_first adds an unlabelled-positive row at the start, listing every news
    an hour before any request."""
    TE._write_validation_dir(d)
    rows = open(os.path.join(d, "behaviors.tsv")).read().splitlines()
    rng = np.random.default_rng(5)
    out = []
    for i, ln in enumerate(rows):
        f = ln.split("\t")
        f[2] = _stamp(1 + int(rng.integers(0, 40)))
        f[4] = " ".join(x for x in f[4].split() if x.split("-")[0] not in ("N0", "N1", "N2") or shown_first)
        out.append("\t".join(f) if f[4] else None)
    out = [x for x in out if x is not None]
    if shown_first:
        out.insert(0, "0\tU3\t" + _stamp(0) + "\t\t" + " ".join(f"N{i}-0" for i in range(TE.N_NEWS)))
    open(os.path.join(d, "behaviors.tsv"), "w").write("\n".join(out) + "\n")


def _coeff(D):
    return 2.0 ** -15 + 3 * ((D + 63) // 64 * 64) * 2.0 ** -23


def _exact(model, d, u2i):
    """Host fp64 restatement: (tables, pad, ids, S, E) with S / E (U, n) the exact scores and the stated bound per line user."""
    from newsrec_b200 import evaluate as E
    from newsrec_b200.recommend import pool_operands
    with torch.no_grad():
        index, matrix = E.news_matrix(model, d)
        t = E.build_tables(d, index, model.config.num_clicked_news_a_user, 10 ** 9, u2i)
        pad = index["PADDED_NEWS"]
        users, dnn = pool_operands(model, t, matrix, E.new_flag(matrix.device))
    pool = matrix[:pad]
    if dnn is None:
        u64, p64 = users.double(), pool.double()
        S, Eb = u64 @ p64.T, _coeff(pool.shape[1]) * (u64.abs() @ p64.abs().T)
    else:
        S, Eb = AR.exact_and_bound(users if users.dim() == 3 else users.unsqueeze(1), pool, dnn, DEV)
    return t, pad, E.read_news(d, [])[0], S.cpu().numpy(), Eb.cpu().numpy()


def _eligible(d, ids, t_req, H):
    """(U or S, n) bool: t - W <= first_shown <= t from a plain loop over behaviors.tsv."""
    from newsrec_b200 import window
    first = {}
    for ln in open(os.path.join(d, "behaviors.tsv")).read().splitlines():
        f = ln.split("\t")
        ts = int(window.parse_times([f[2]])[0])
        for x in f[4].split():
            nid = x.split("-")[0]
            first[nid] = min(first.get(nid, ts), ts)
    fs = np.array([first.get(x, np.nan) for x in ids], np.float64)
    W = H * HOUR
    return (fs[None, :] >= np.asarray(t_req, np.float64)[:, None] - W) & (fs[None, :] <= np.asarray(t_req, np.float64)[:, None])


@pytest.mark.parametrize("name", ["NRMS", "HiFiArk"])
def test_recommend_and_pool_eval_with_a_window(name, tmp_path):
    from newsrec_b200 import evaluate as E
    from newsrec_b200 import pool_eval as P
    from newsrec_b200 import window
    from newsrec_b200.recommend import recommend
    d = str(tmp_path)
    _write_timed_split(d)
    u2i = os.path.join(d, "user2int.tsv")
    model = _model(name).eval()
    H, k = 6, 20
    t, pad, ids, S, Eb = _exact(model, d, u2i)
    beh = E.read_behaviors(d)
    times = window.parse_times(beh["time"])
    # recommend: the lines within the per-pair bound of the fp64 restatement, the same file at chunk 7 and one chunk
    files = [str(tmp_path / f"rec{c}.tsv") for c in (7, 10 ** 9)]
    for c, f in zip((7, 10 ** 9), files):
        recommend(model, d, f, k, user2int_path=u2i, chunk_users=c, max_age_hours=H)
    assert open(files[0], "rb").read() == open(files[1], "rb").read()
    lines = [ln.split("\t")[1] for ln in open(files[0]).read().splitlines()]
    elig_u = _eligible(d, ids, times[E.distinct_histories(beh).index.to_numpy()], H)
    assert not elig_u[:, :3].any()  # never listed: in no window
    tol = 2 * Eb + 1e-6 * np.abs(S)
    for u, line in enumerate(lines):
        rows = [ids.index(x) for x in line.split(",")] if line else []
        elig = elig_u[u].copy()
        elig[[r for r in t.history[u] if r != pad]] = False
        assert all(elig[r] for r in rows) and len(rows) == min(k, int(elig.sum()))
        cand = np.sort(S[u, elig])[::-1]
        kth = cand[len(rows) - 1] if elig.sum() >= k else -np.inf
        for j, r in enumerate(rows):
            assert S[u, r] >= kth - tol[u, r]
            if j + 1 < len(rows):
                assert S[u, r] >= S[u, rows[j + 1]] - tol[u, r] - tol[u, rows[j + 1]]
    # evaluate_pool: every rank within the band over the impression's window, the JSON's window figures, chunk invariance
    res = [P.evaluate_pool(model, d, (1, 5, 20), user2int_path=u2i, chunk_impressions=c, max_age_hours=H) for c in (7, 10 ** 9)]
    assert res[0] == res[1]
    win = window.load("evaluate_pool", d, H)
    imp, rows, offsets, rank, score, w = P._positions(model, d, win, True, 10 ** 9, u2i, 7)
    elig_i = _eligible(d, ids, times[imp], H)
    assert res[0]["pool_size_mean"] == float(np.mean(elig_i.sum(1)))
    outside = 0
    for s_ in range(len(imp)):
        u = int(t.seg_user[imp[s_]])
        P_i = rows[offsets[s_]:offsets[s_ + 1]]
        outside += int((~elig_i[s_, P_i]).sum())
        el = elig_i[s_].copy()
        el[[r for r in t.history[u] if r != pad]] = False
        el[P_i] = False
        for j, p in enumerate(P_i):
            dlt, e = S[u] - S[u, p], Eb[u] + Eb[u, p]
            lo, hi = int((el & (dlt > e)).sum()), int((el & (dlt >= -e)).sum())
            assert lo <= rank[offsets[s_] + j] <= hi, (s_, p, lo, rank[offsets[s_] + j], hi)
    assert res[0]["targets_outside_window"] == outside and res[0]["max_age_hours"] == H
    # evaluate_lists: chunk invariance, coverage over the news eligible somewhere
    lres = [P.evaluate_lists(model, d, 10, user2int_path=u2i, chunk_impressions=c, max_age_hours=H) for c in (7, 10 ** 9)]
    assert lres[0] == lres[1] and lres[0]["n_pool"] == int(elig_i.any(0).sum())
    assert lres[0]["targets_outside_window"] == outside
    # a window that holds every shown news: evaluate_lists' plain lists agree with evaluate_pool when nothing is excluded
    inf_lists = P.evaluate_lists(model, d, 20, (1, 5, 20), exclude_clicked=False, user2int_path=u2i, max_age_hours=float("inf"))
    inf_pool = P.evaluate_pool(model, d, (1, 5, 20), exclude_clicked=False, user2int_path=u2i, max_age_hours=float("inf"))
    assert inf_pool["targets_outside_window"] == 0
    for K in (1, 5, 20):
        assert inf_lists[f"recall@{K}"] == inf_pool[f"recall@{K}"] and inf_lists[f"ndcg@{K}"] == inf_pool[f"ndcg@{K}"]


@pytest.mark.parametrize("name", ["NRMS", "DKN"])
def test_an_infinite_window_over_news_shown_before_every_request_is_the_plain_output(name, tmp_path):
    from newsrec_b200 import pool_eval as P
    from newsrec_b200.recommend import recommend
    d = str(tmp_path)
    _write_timed_split(d, shown_first=True)
    u2i = os.path.join(d, "user2int.tsv")
    model = _model(name).eval()
    a, b = str(tmp_path / "plain.tsv"), str(tmp_path / "inf.tsv")
    recommend(model, d, a, 20, user2int_path=u2i)
    recommend(model, d, b, 20, user2int_path=u2i, max_age_hours=float("inf"), chunk_users=7)
    assert open(a, "rb").read() == open(b, "rb").read()
    plain = P.evaluate_pool(model, d, (1, 5, 20), user2int_path=u2i)
    inf = P.evaluate_pool(model, d, (1, 5, 20), user2int_path=u2i, max_age_hours=float("inf"))
    assert {x: inf[x] for x in plain} == plain and inf["pool_size_mean"] == TE.N_NEWS
    plain = P.evaluate_lists(model, d, 10, user2int_path=u2i)
    inf = P.evaluate_lists(model, d, 10, user2int_path=u2i, max_age_hours=float("inf"), chunk_impressions=7)
    assert {x: inf[x] for x in plain} == plain and inf["n_pool"] == TE.N_NEWS
