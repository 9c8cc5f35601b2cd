"""Recommendation over the whole pool on the H100: nr_topk_dot / ops.top_k_scores against an fp64 brute force on the same fp32
inputs, then newsrec_b200.recommend end to end against predict's ranks and a host recompute, independent of the chunk size.

Bound: each returned score is within e_un = (2^-15 + 3 round_up(D, 64) 2^-23) sum_i |u_i||n_i| of the fp64 dot product, the
bound include/newsrec_b200.h states for the hi/lo planes (the dropped lo.lo term and the plane roundings: 2^-15; the fp32
tensor-core accumulation of 3 round_up(D, 64) products: 3 round_up(D, 64) 2^-23).  Set and order follow from it: a news
whose fp64 score beats the fp64 k-th best by more than 2e must be returned, and a returned news is within 2e of it."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import gpu_checks as G
import test_gpu_evaluate as TE

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def _bound_coeff(D):
    return 2.0 ** -15 + 3 * ((D + 63) // 64 * 64) * 2.0 ** -23


def _csr(lists):
    offs = np.zeros(len(lists) + 1, np.int64)
    offs[1:] = np.cumsum([len(x) for x in lists])
    rows = np.concatenate([np.asarray(x, np.int64) for x in lists]) if offs[-1] else np.zeros(0, np.int64)
    return torch.from_numpy(rows), torch.from_numpy(offs)


def _check(users, news, k, excl=None):
    """Runs ops.top_k_scores and checks score bound, set, order and padding against fp64; returns (idx, score)."""
    from newsrec_b200.ops import top_k_scores
    rows, offs = _csr(excl) if excl is not None else (None, None)
    idx, score = top_k_scores(users, news, k, rows, offs)
    U, n, D = users.shape[0], news.shape[0], users.shape[1]
    assert idx.shape == (U, k) and score.shape == (U, k)
    u64, n64 = users.double().to(DEV), news.double().to(DEV)
    S = u64 @ n64.T
    E = _bound_coeff(D) * (u64.abs() @ n64.abs().T)
    elig = torch.ones((U, n), dtype=torch.bool, device=DEV)
    if excl is not None:
        for u, lst in enumerate(excl):
            if len(lst):
                elig[u, torch.as_tensor(np.asarray(lst, np.int64), device=DEV)] = False
    n_elig = elig.sum(1)
    idx_c, score_c = idx.to(DEV), score.to(DEV)
    live = idx_c >= 0
    want = torch.minimum(n_elig, torch.tensor(k, device=DEV))
    assert torch.equal(live.sum(1), want), "number of returned news"
    assert torch.equal(live, torch.arange(k, device=DEV)[None, :] < want[:, None]), "live slots first"
    assert bool((score_c[~live] == float("-inf")).all()), "padding scores"
    r = idx_c.clamp(min=0)
    s_ref = torch.gather(S, 1, r)
    e_ref = torch.gather(E, 1, r)
    assert bool(((score_c.double() - s_ref).abs() <= e_ref)[live].all()), "score bound"
    assert bool(torch.gather(elig, 1, r)[live].all()), "an excluded news was returned"
    # distinct rows
    srt = torch.sort(torch.where(live, idx_c, torch.full_like(idx_c, -1) - torch.arange(k, device=DEV)), dim=1).values
    assert bool((srt[:, 1:] != srt[:, :-1]).all()), "a row returned twice"
    # order: non-increasing, ties by row
    if k > 1:
        a, b = score_c[:, :-1], score_c[:, 1:]
        both = live[:, :-1] & live[:, 1:]
        assert bool((a >= b)[both].all()), "scores not non-increasing"
        assert bool(((a != b) | (idx_c[:, :-1] < idx_c[:, 1:]))[both].all()), "equal scores not in row order"
    # set: against the fp64 k-th best of the eligible news
    Sm = torch.where(elig, S, torch.tensor(float("-inf"), dtype=torch.float64, device=DEV))
    kk = min(k, n)
    kth = torch.topk(Sm, kk, dim=1).values[:, -1]
    full = n_elig >= k
    kth = torch.where(full, kth, torch.tensor(float("-inf"), dtype=torch.float64, device=DEV))
    must = elig & (S > kth[:, None] + 2 * E)
    got = torch.zeros((U, n), dtype=torch.int32, device=DEV).scatter_add_(1, r, live.int()) > 0
    assert bool((got | ~must).all()), "a news clearly above the k-th best is missing"
    assert bool(((s_ref >= kth[:, None] - 2 * e_ref) | ~live).all()), "a returned news is clearly below the k-th best"
    return idx, score


CASES = [  # (n_users, n_news, D, k)
    (1, 1, 300, 1), (63, 127, 300, 10), (64, 4097, 400, 100), (65, 9, 150, 10), (1100, 4097, 300, 10),
    (1000, 30_000, 300, 128), (65, 30_000, 400, 100), (64, 127, 150, 128), (63, 99, 300, 100), (1, 30_000, 150, 1),
]


@pytest.mark.parametrize("U,n,D,k", CASES)
def test_top_k_matches_fp64(U, n, D, k):
    g = torch.Generator().manual_seed(U * 7 + n + D + k)
    users = torch.randn(U, D, generator=g)
    news = torch.randn(n, D, generator=g)
    _check(users, news, k)


def test_fewer_eligible_than_k_and_all_negative():
    g = torch.Generator().manual_seed(1)
    D = 300
    users = torch.randn(70, D, generator=g)
    news = torch.randn(127, D, generator=g)
    news_neg = -users[0].abs().sign()[None, :] * torch.rand(50, D, generator=g)  # all scores of user 0 negative
    for k in (128, 100):
        idx, _ = _check(users, news, k)
        assert (idx[:, :127] >= 0).all() and (idx[:, 127:] == -1).all()
    pos = users.abs()
    _check(pos, -torch.rand(9, D, generator=g), 10)  # every score negative, fewer news than k
    _check(users[:1], news_neg, 10)


def test_exclusions_empty_longer_than_k_and_whole_pool():
    g = torch.Generator().manual_seed(2)
    U, n, D = 66, 4097, 300
    users = torch.randn(U, D, generator=g)
    news = torch.randn(n, D, generator=g)
    rng = np.random.default_rng(2)
    excl = []
    for u in range(U):
        if u % 3 == 0:
            excl.append([])
        elif u % 3 == 1:  # longer than k, unsorted, with duplicates
            lst = rng.integers(0, n, 300)
            excl.append(np.concatenate([lst, lst[:20]]))
        else:  # the user's own best 40 news, so that the exclusion changes the answer
            s = (users[u:u + 1].double() @ news.double().T)[0]
            excl.append(torch.topk(s, 40).indices.numpy()[::-1].copy())
    _check(users, news, 10, excl)
    _check(users, news, 128, excl)
    small = news[:300]
    everything = [np.arange(300)] * 5
    idx, score = _check(users[:5], small, 10, everything)
    assert (idx == -1).all() and (score == float("-inf")).all()
    _check(users[:5], small, 10, [np.arange(295)] * 5)  # 5 eligible news left, k = 10


def test_duplicates_and_near_ties_keep_row_order():
    g = torch.Generator().manual_seed(3)
    D, n, k = 300, 5000, 10
    users = torch.randn(65, D, generator=g)
    news = torch.randn(n, D, generator=g)
    best = torch.topk(users[0:1] @ news.T, 1).indices.item()
    for r in (7, 1234, 4999):  # identical copies of user 0's best news
        news[r] = news[best]
    # a cluster of nearly equal news straddling user 1's k-th place
    base = news[100] * 0 + users[1] / users[1].norm() * 3.0
    for j in range(20):
        news[2000 + 37 * j] = base + 1e-6 * torch.randn(D, generator=g)
    idx, score = _check(users, news, k)
    rows0 = idx[0].tolist()
    dup = sorted({best, 7, 1234, 4999})
    assert rows0[:4] == dup, rows0
    assert (score[0, :4] == score[0, 0]).all()


def test_determinism_and_flags():
    from newsrec_b200 import launch_count
    from newsrec_b200.ops import top_k_scores
    g = torch.Generator().manual_seed(4)
    users = torch.randn(300, 400, generator=g)
    news = torch.randn(20_000, 400, generator=g)
    a = top_k_scores(users, news, 100)
    b = top_k_scores(users, news, 100)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1].view(torch.int32), b[1].view(torch.int32))
    few = top_k_scores(users[:3], news, 100)  # several splits + the merge launch: the same answer
    assert torch.equal(few[0], a[0][:3]) and torch.equal(few[1], a[1][:3])
    rows, offs = _csr([[5], [20_000], []])
    with pytest.raises(IndexError, match="outside the news pool"):
        top_k_scores(users[:3], news, 10, rows, offs)
    bad = news.clone()
    bad[777, 3] = float("nan")
    with pytest.raises(ValueError, match="not finite"):
        top_k_scores(users[:3], bad, 10)
    n0 = launch_count()
    i0, s0 = top_k_scores(users[:0], news, 10)
    i1, s1 = top_k_scores(users[:4], news[:0], 10)
    assert launch_count() == n0
    assert i0.shape == (0, 10) and (i1 == -1).all() and (s1 == float("-inf")).all()


def test_refused_before_any_launch():
    from newsrec_b200 import NewsrecError, launch_count
    from newsrec_b200.ops import top_k_scores
    users, news = torch.randn(4, 30), torch.randn(50, 30)
    n0 = launch_count()
    for k in (0, 129, -1, 2.0):
        with pytest.raises(NewsrecError, match="k="):
            top_k_scores(users, news, k)
    with pytest.raises(NewsrecError):
        top_k_scores(users, torch.randn(50, 31), 10)
    assert launch_count() == n0


def test_guard_bands_of_the_raw_entry_point():
    from newsrec_b200 import load_library
    lib = load_library()
    g = torch.Generator().manual_seed(5)
    U, n, D, k = 70, 3000, 150, 100
    users = torch.randn(U, D, generator=g).to(DEV)
    news = torch.randn(n, D, generator=g).to(DEV)
    ws_bytes = int(lib.nr_topk_dot_workspace(U, n, D, k))
    assert ws_bytes > 0 and lib.nr_topk_dot_workspace(U, n, D, 129) == -1
    idx = G._Guarded(U * k, torch.int64, -777, sentinel=-4242)
    score = G._Guarded(U * k, torch.float32, float("nan"))
    ws = G._Guarded(ws_bytes + 256, torch.uint8, 0xAB, sentinel=0x5C)
    flags = G._Guarded(2, torch.int32, 0, sentinel=-3)
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    wp = ws.all.data_ptr()
    pad = (-wp) % 256
    rc = lib.nr_topk_dot(users.data_ptr(), U, D, news.data_ptr(), n, D, D, k, None, None, idx.all.data_ptr(),
                         score.all.data_ptr(), flags.all.data_ptr(), flags.all.data_ptr() + 4, wp + pad, ws_bytes, s)
    assert rc == 0
    torch.cuda.synchronize()
    assert idx.guard_ok() and score.guard_ok() and flags.guard_ok() and ws.guard_ok()
    assert not torch.isnan(score.body).any() and (idx.body >= 0).all()
    assert (flags.body == 0).all()
    # refused shapes leave everything untouched
    for bad in [dict(k=0), dict(k=129), dict(D=0), dict(ld=D - 1), dict(ws=ws_bytes - 1)]:
        before = (idx.body.clone(), score.body.clone())
        rc = lib.nr_topk_dot(users.data_ptr(), U, bad.get("ld", D), news.data_ptr(), n, D, bad.get("D", D), bad.get("k", k),
                             None, None, idx.all.data_ptr(), score.all.data_ptr(), flags.all.data_ptr(),
                             flags.all.data_ptr() + 4, wp + pad, bad.get("ws", ws_bytes), s)
        assert rc == -1 and lib.nr_last_error().decode().startswith("nr_topk_dot"), bad
        torch.cuda.synchronize()
        assert torch.equal(idx.body, before[0]) and G._bits_equal(score.body, before[1])


# ------------------------------------------------------------------------------------------------------------------------
# end to end
# ------------------------------------------------------------------------------------------------------------------------
FAMILIES = {"NRMS": "nrms", "LSTUR": "lstur_ini", "NAML": "naml"}


def _model(name):
    torch.manual_seed(0)
    model, cfg = G.build_model(FAMILIES[name], V=TE.V, ncat=TE.NCAT, nusers=TE.NUSERS, H=TE.H)
    cfg.batch_size = 2
    return model.eval()


def _read(path):
    out = []
    for ln in open(path, "rb").read().decode().splitlines():
        u, rest = ln.split("\t")
        out.append((u, rest.split(",") if rest else []))
    return out


@pytest.mark.parametrize("name", list(FAMILIES))
def test_recommend_matches_predict_and_a_host_recompute(name, tmp_path):
    from newsrec_b200 import evaluate as E
    from newsrec_b200.ops import top_k_scores
    from newsrec_b200.predict import build_prediction_tables, predict
    from newsrec_b200.recommend import recommend
    d = str(tmp_path)
    TE._write_validation_dir(d)
    u2i = os.path.join(d, "user2int.tsv")
    model = _model(name)
    k = 20
    files = {}
    for chunk in (1, 7, 10 ** 9):
        files[chunk] = str(tmp_path / f"rec_{chunk}.tsv")
        n_lines = recommend(model, d, files[chunk], k, user2int_path=u2i, chunk_users=chunk)
        assert not os.path.exists(files[chunk] + ".partial")
    data = {c: open(f, "rb").read() for c, f in files.items()}
    assert data[1] == data[7] == data[10 ** 9]
    lines = _read(files[1])
    assert len(lines) == n_lines
    with torch.no_grad():
        index, matrix = E.news_matrix(model, d)
        beh = E.read_behaviors(d)
        user, history, length, hist_row = E.user_tables(beh, index, model.config.num_clicked_news_a_user, u2i)
        uv = E.user_vectors(model, E.build_tables(d, index, model.config.num_clicked_news_a_user, 10 ** 9, u2i), matrix,
                            E.new_flag(matrix.device))
    assert [u for u, _ in lines] == E.distinct_histories(beh)["user"].tolist()
    pad = index["PADDED_NEWS"]
    ids = E.read_news(d, [])[0]
    S = uv.double() @ matrix[:pad].double().T
    Eb = _bound_coeff(matrix.shape[1]) * (uv.double().abs() @ matrix[:pad].double().abs().T)
    for u, (_, got) in enumerate(lines):
        hist = set(int(r) for r in history[u] if r != pad)
        rows = [ids.index(x) for x in got]
        assert not hist & set(rows)
        elig = [r for r in range(pad) if r not in hist]
        assert len(rows) == min(k, len(elig))
        s = S[u, elig]
        kth = torch.sort(s, descending=True).values[len(rows) - 1] if len(elig) >= k else float("-inf")
        for r in rows:
            assert S[u, r] >= kth - 2 * Eb[u, r]
        for j in range(len(rows) - 1):
            assert S[u, rows[j]] >= S[u, rows[j + 1]] - 2 * (Eb[u, rows[j]] + Eb[u, rows[j + 1]])
    # one impression's candidates only, k = its size: predict's order
    out = str(tmp_path / "prediction.txt")
    predict(model, d, out, user2int_path=u2i)
    t = build_prediction_tables(d, index, model.config.num_clicked_news_a_user, u2i)
    pred = open(out).read().splitlines()
    checked = 0
    for s_ in range(len(t.seg_user)):
        a, b = t.seg_offsets[s_], t.seg_offsets[s_ + 1]
        cand = torch.from_numpy(t.cand[a:b])
        if b - a > 128 or len(set(t.cand[a:b].tolist())) != b - a:
            continue
        u = int(hist_row[beh["clicked_news"].iloc[s_]])
        idx, score = top_k_scores(uv[u:u + 1], matrix[cand.to(DEV)], int(b - a))
        ranks = [int(x) for x in pred[s_].split(" ", 1)[1][1:-1].split(",")]
        order_pred = np.argsort(ranks, kind="stable")  # candidate positions, best first
        sc = (uv[u:u + 1].double() @ matrix[cand.to(DEV)].double().T)[0].cpu().numpy()
        eb = (_bound_coeff(matrix.shape[1]) * (uv[u:u + 1].double().abs() @ matrix[cand.to(DEV)].double().abs().T))[0].cpu().numpy()
        got = idx[0].cpu().numpy()
        for p_, q_ in zip(got, order_pred):
            assert p_ == q_ or abs(sc[p_] - sc[q_]) <= 2 * (eb[p_] + eb[q_]) + 1e-6 * abs(sc[q_]), (s_, got, order_pred)
        checked += 1
    assert checked >= 50


def test_recommend_memory_is_bounded_by_the_chunk(tmp_path):
    from newsrec_b200.recommend import recommend
    d = str(tmp_path)
    TE._write_validation_dir(d)
    u2i = os.path.join(d, "user2int.tsv")
    model = _model("NRMS")
    peaks = []
    for rep in (1, 8):  # the same users repeated: 8x the lines
        if rep > 1:
            src = open(os.path.join(d, "behaviors.tsv")).read().splitlines()
            with open(os.path.join(d, "behaviors.tsv"), "w") as f:
                for r in range(rep):
                    for ln in src:
                        c = ln.split("\t")
                        c[3] = c[3] + f" N{r}" if c[3] else f"N{r}"  # distinct histories per copy
                        f.write("\t".join(c) + "\n")
        recommend(model, d, str(tmp_path / "warm.tsv"), 10, user2int_path=u2i, chunk_users=4)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        n = recommend(model, d, str(tmp_path / f"rec{rep}.tsv"), 10, user2int_path=u2i, chunk_users=4)
        torch.cuda.synchronize()
        peaks.append((n, torch.cuda.max_memory_allocated()))
    assert peaks[1][0] > 4 * peaks[0][0]
    assert peaks[1][1] <= peaks[0][1] + (1 << 20), peaks


def test_recommend_non_finite_score_raises_and_leaves_no_file(tmp_path, monkeypatch):
    from newsrec_b200 import recommend as R
    d = str(tmp_path)
    TE._write_validation_dir(d)
    model = _model("NRMS")
    orig, calls = R.user_vectors, []

    def poisoned(*a, **k):
        v = orig(*a, **k)
        calls.append(1)
        if len(calls) == 2:
            v[-1, 0] = float("nan")
        return v

    monkeypatch.setattr(R, "user_vectors", poisoned)
    out = str(tmp_path / "rec.tsv")
    with pytest.raises(ValueError, match="not finite"):
        R.recommend(model, d, out, 10, user2int_path=os.path.join(d, "user2int.tsv"), chunk_users=3)
    assert not os.path.exists(out) and not os.path.exists(out + ".partial")
