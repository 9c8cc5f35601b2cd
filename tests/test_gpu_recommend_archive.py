"""Recommendation over the whole pool under Hi-Fi Ark's and DKN's DNN click score on the H100: nr_topk_archive /
ops.top_k_scores(..., dnn=) against the fp64 restatement and the stated bound of tests/archive_pool_ref.py, exactly against
the kernel's own score bits, and newsrec_b200.recommend end to end for both families."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import archive_pool_ref as AR
import test_gpu_evaluate as TE
from test_gpu_predict import _model

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)

SHAPES = [(5, 300, 24), (1, 150, 17), (1, 4, 1), (32, 400, 32), (3, 52, 11)]  # (P, F, hidden)


def _csr(lists):
    offs = np.zeros(len(lists) + 1, np.int64)
    offs[1:] = np.cumsum([len(x) for x in lists])
    rows = np.concatenate([np.asarray(x, np.int64) for x in lists]) if offs[-1] else np.zeros(0, np.int64)
    return torch.from_numpy(rows), torch.from_numpy(offs)


def _users(A):
    return A[:, 0] if A.shape[1] == 1 else A  # P = 1 goes in as (U, F), as DKN's user vectors do


def _check(A, C_, dnn, k, excl=None):
    """ops.top_k_scores(..., dnn=) checked as test_gpu_recommend._check checks the dot scorer; returns (idx, score)."""
    from newsrec_b200.ops import top_k_scores
    rows, offs = _csr(excl) if excl is not None else (None, None)
    idx, score = top_k_scores(_users(A), C_, k, rows, offs, dnn=dnn)
    U, n = A.shape[0], C_.shape[0]
    assert idx.shape == (U, k) and score.shape == (U, k)
    S, E = AR.exact_and_bound(A, C_, dnn, DEV)
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
    s_ref, e_ref = torch.gather(S, 1, r), torch.gather(E, 1, r)
    assert bool(((score_c.double() - s_ref).abs() <= e_ref)[live].all()), \
        float(((score_c.double() - s_ref).abs() / e_ref)[live].max())
    assert bool(torch.gather(elig, 1, r)[live].all()), "an excluded news was returned"
    srt = torch.sort(torch.where(live, idx_c, torch.full_like(idx_c, -1) - torch.arange(k, device=DEV)), dim=1).values
    assert bool((srt[:, 1:] != srt[:, :-1]).all()), "a row returned twice"
    if k > 1:
        a, b = score_c[:, :-1], score_c[:, 1:]
        both = live[:, :-1] & live[:, 1:]
        assert bool((a >= b)[both].all()), "scores not non-increasing"
        assert bool(((a != b) | (idx_c[:, :-1] < idx_c[:, 1:]))[both].all()), "equal scores not in row order"
    Sm = torch.where(elig, S, torch.tensor(float("-inf"), dtype=torch.float64, device=DEV))
    kth = torch.topk(Sm, min(k, n), dim=1).values[:, -1]
    kth = torch.where(n_elig >= k, kth, torch.tensor(float("-inf"), dtype=torch.float64, device=DEV))
    must = elig & (S > kth[:, None] + 2 * E)
    got = torch.zeros((U, n), dtype=torch.int32, device=DEV).scatter_add_(1, r, live.int()) > 0
    assert bool((got | ~must).all()), "a news clearly above the k-th best is missing"
    assert bool(((s_ref >= kth[:, None] - 2 * e_ref) | ~live).all()), "a returned news is clearly below the k-th best"
    return idx, score


def _cases():
    for P, F, hid in SHAPES:
        G = 64 // P
        for U, n, k in ((1, 1, 1), (G, 63, 10), (G + 1, 64, 128), (200, 65, 10), (G + 1, 5000, 128), (200, 5000, 10),
                        (1, 5000, 1)):
            yield P, F, hid, U, n, k


@pytest.mark.parametrize("P,F,hid,U,n,k", list(_cases()))
def test_top_k_matches_fp64(P, F, hid, U, n, k):
    g = torch.Generator().manual_seed(P * 1000 + F + hid + U + n + k)
    A, C_, dnn = AR.operands(g, U, P, F, hid, n)
    rng = np.random.default_rng(U + n)
    excl = [[] if u % 3 == 0 else rng.integers(0, n, size=int(rng.integers(1, 2 * k + 2))).tolist() for u in range(U)]
    _check(A, C_, dnn, k, excl)


@pytest.mark.parametrize("P,F,hid", SHAPES)
def test_agrees_with_the_impression_scorer(P, F, hid):
    """nr_archive_score_fwd (evaluate()'s scorer) on every pair of the pool agrees within twice the bound."""
    from newsrec_b200.ops import top_k_scores
    from newsrec_b200.ops_hifiark import score_impressions
    U, n = 9, 100
    g = torch.Generator().manual_seed(P + F)
    A, C_, dnn = AR.operands(g, U, P, F, hid, n)
    if F % 4:  # the impression scorer takes F % 4 == 0 (DKN's widened rows): pad with zero columns, which change nothing
        pad = 4 - F % 4
        Cw = torch.nn.functional.pad(C_, (0, pad))
        Aw = torch.nn.functional.pad(A, (0, pad))
        W1 = dnn[0]
        W1w = torch.cat([torch.nn.functional.pad(W1[:, :F], (0, pad)), torch.nn.functional.pad(W1[:, F:], (0, pad))], 1)
        fw = (Cw, Aw, (W1w,) + tuple(dnn[1:]))
    else:
        fw = (C_, A, dnn)
    cand = torch.arange(n, device=DEV).repeat(U)
    seg = torch.arange(0, U * n + 1, n, device=DEV)
    flag = torch.zeros(1, dtype=torch.int32, device=DEV)
    ref = score_impressions(fw[0].to(DEV), cand, seg, fw[1].to(DEV), *(t.to(DEV) for t in fw[2]), flag).view(U, n).double()
    idx, score = top_k_scores(_users(A), C_, n, dnn=dnn)
    _, E = AR.exact_and_bound(A, C_, dnn, DEV)
    r = idx.to(DEV)
    assert bool(((score.double().to(DEV) - torch.gather(ref, 1, r)).abs() <= 2 * torch.gather(E, 1, r)).all())


def _all_scores(A, C_, dnn):
    """Every pair's kernel score, (U, n) fp32, from k = n <= 128 (the list holds the whole pool)."""
    from newsrec_b200.ops import top_k_scores
    n = C_.shape[0]
    idx, score = top_k_scores(_users(A), C_, n, dnn=dnn)
    out = torch.empty_like(score)
    out.scatter_(1, idx.to(out.device), score)
    return out, idx, score


@pytest.mark.parametrize("P,F,hid", SHAPES)
def test_cap_mmr_and_bits_against_the_kernels_own_scores(P, F, hid):
    from newsrec_b200.ops import top_k_scores
    U, n = 70, 120
    g = torch.Generator().manual_seed(3 * P + F)
    A, C_, dnn = AR.operands(g, U, P, F, hid, n)
    cats = torch.randint(0, 6, (n,), generator=g).int()
    allsc, idx_all, sc_all = _all_scores(A, C_, dnn)
    for k, m in ((10, 2), (40, 3), (120, 1)):
        idx, score = top_k_scores(_users(A), C_, k, dnn=dnn, categories=cats, max_per_category=m)
        idx, score = idx.cpu().numpy(), score.cpu().numpy()
        for u in range(U):
            taken = AR.capped_walk(sc_all[u].cpu().numpy(), idx_all[u].cpu().numpy(), cats.numpy(), k, m)
            assert idx[u, :len(taken)].tolist() == [r for _, r in taken]
            assert np.array_equal(score[u, :len(taken)], np.array([s for s, _ in taken], np.float32))
            assert (idx[u, len(taken):] == -1).all() and (score[u, len(taken):] == -np.inf).all()
        plain = top_k_scores(_users(A), C_, k, dnn=dnn)
        capk = top_k_scores(_users(A), C_, k, dnn=dnn, categories=cats, max_per_category=k)
        assert torch.equal(plain[0], capk[0]) and torch.equal(plain[1], capk[1]), "m >= k is the plain list"
        mmr = top_k_scores(_users(A), C_, k, dnn=dnn, mmr_lambda=1.0, mmr_depth=min(128, 2 * k))
        assert torch.equal(plain[0], mmr[0]) and torch.equal(plain[1], mmr[1]), "MMR at lambda 1 is the plain list"
        assert torch.equal(plain[0], idx_all[:, :k]) and torch.equal(plain[1], sc_all[:, :k])
    div = top_k_scores(_users(A), C_, 10, dnn=dnn, mmr_lambda=0.3)
    assert (div[0] >= 0).all()


@pytest.mark.parametrize("P,F,hid", [(5, 300, 24), (1, 150, 17), (3, 52, 11)])
def test_bits_do_not_depend_on_users_chunks_or_splits(P, F, hid):
    from newsrec_b200.ops import top_k_scores
    U, n, k = 1500, 1000, 16
    g = torch.Generator().manual_seed(P + 11)
    A, C_, dnn = AR.operands(g, U, P, F, hid, n)
    base = top_k_scores(_users(A), C_, k, dnn=dnn)
    again = top_k_scores(_users(A), C_, k, dnn=dnn)
    assert torch.equal(base[0], again[0]) and torch.equal(base[1], again[1]), "two runs"
    perm = torch.randperm(U, generator=g)
    pi, ps = top_k_scores(_users(A[perm]), C_, k, dnn=dnn)
    assert torch.equal(pi, base[0][perm.to(pi.device)]) and torch.equal(ps, base[1][perm.to(ps.device)]), "permuted users"
    for chunk in (1, 7, 100):  # fewer CTAs: more splits of the pool
        parts = [top_k_scores(_users(A[a:min(a + chunk, 300)]), C_, k, dnn=dnn) for a in range(0, 300, chunk)]
        assert torch.equal(torch.cat([p[0] for p in parts]), base[0][:300]), chunk
        assert torch.equal(torch.cat([p[1] for p in parts]), base[1][:300]), chunk


def test_flags_raise():
    from newsrec_b200.ops import top_k_scores
    g = torch.Generator().manual_seed(5)
    A, C_, dnn = AR.operands(g, 20, 5, 300, 24, 200)
    rows, offs = _csr([[3, 1000]] + [[]] * 19)
    with pytest.raises(IndexError):
        top_k_scores(A, C_, 10, rows, offs, dnn=dnn)
    bad = A.clone()
    bad[7, 2, 5] = float("nan")
    with pytest.raises(ValueError, match="not finite"):
        top_k_scores(bad, C_, 10, dnn=dnn)
    bad = A[:, :1].clone()
    bad[3, 0, 0] = float("inf")
    with pytest.raises(ValueError, match="not finite"):
        top_k_scores(bad[:, 0], C_, 10, dnn=(torch.randn(24, 600, generator=g),) + dnn[1:])


def test_raw_entry_points_refuse_every_limit_before_a_launch():
    import newsrec_b200
    lib = newsrec_b200.load_library()
    buf = torch.zeros(1 << 16, dtype=torch.float32, device=DEV)
    ws = torch.zeros(1 << 20, dtype=torch.uint8, device=DEV)
    p, wsp = C.c_void_p(buf.data_ptr()), C.c_void_p(ws.data_ptr())
    good = dict(U=4, P=5, n=10, F=8, hid=4, k=3)
    bad = [dict(P=0), dict(P=33), dict(hid=0), dict(hid=33), dict(F=0), dict(F=4097), dict(k=0), dict(k=129),
           dict(U=-1), dict(U=(2 ** 31 - 64) // 5), dict(n=-1), dict(n=2 ** 31 - 64)]
    before = newsrec_b200.launch_count()
    for over in bad:
        a = {**good, **over}
        assert lib.nr_topk_archive_workspace(a["U"], a["P"], a["n"], a["F"], a["hid"], a["k"]) == -1, over
        assert lib.nr_topk_archive(p, a["U"], a["P"], p, a["n"], a["F"], p, p, a["hid"], p, p, a["k"], None, None, None, 0,
                                   p, p, p, p, wsp, ws.numel(), None) == -1, over
        if "k" not in over:
            assert lib.nr_pool_ranks_archive_workspace(a["U"], a["P"], a["n"], a["F"], a["hid"]) == -1, over
            assert lib.nr_pool_ranks_archive(p, a["U"], a["P"], p, a["n"], a["F"], p, p, a["hid"], p, p, p, p, None, None,
                                             p, p, p, p, p, wsp, ws.numel(), None) == -1, over
    a = good
    assert lib.nr_pool_ranks_archive_workspace(a["U"], a["P"], 0, a["F"], a["hid"]) == -1  # ranks need a pool
    assert lib.nr_topk_archive(p, a["U"], a["P"], p, a["n"], a["F"], p, p, a["hid"], p, p, a["k"], None, None, p, 0,
                               p, p, p, p, wsp, ws.numel(), None) == -1  # a cap below 1
    assert lib.nr_topk_archive(None, a["U"], a["P"], p, a["n"], a["F"], p, p, a["hid"], p, p, a["k"], None, None, None, 0,
                               p, p, p, p, wsp, ws.numel(), None) == -1  # a null operand
    assert lib.nr_topk_archive(p, a["U"], a["P"], p, a["n"], a["F"], p, p, a["hid"], p, p, a["k"], None, None, None, 0,
                               p, p, p, p, wsp, 16, None) == -1  # a short workspace
    assert newsrec_b200.launch_count() == before


# ------------------------------------------------------------------------------------------------------------------------
# end to end
# ------------------------------------------------------------------------------------------------------------------------
def _read(path):
    out = []
    for ln in open(path, "rb").read().decode().splitlines():
        u, rest = ln.split("\t")
        out.append((u, rest.split(",") if rest else []))
    return out


def _host_scores(model, d, u2i):
    """(lines' users, history, pad, ids, S (U, n) fp64 host recompute from model.get_prediction) for a whole pool."""
    from newsrec_b200 import evaluate as E
    with torch.no_grad():
        index, matrix = E.news_matrix(model, d)
        beh = E.read_behaviors(d)
        user, history, length, _ = E.user_tables(beh, index, model.config.num_clicked_news_a_user, u2i)
        pad = index["PADDED_NEWS"]
        S = []
        for u in range(len(user)):
            hist = matrix[torch.from_numpy(history[u])].unsqueeze(0)
            uv = model.get_user_vector(hist)[0]
            S.append(model.get_prediction(matrix[:pad], uv).double())
        return E.distinct_histories(beh)["user"].tolist(), history, pad, E.read_news(d, [])[0], torch.stack(S), matrix


def _bound(model, matrix, history, pad):
    """The stated bound of every (user, pool news) pair, from the model's own operands."""
    from newsrec_b200 import evaluate as E
    from newsrec_b200.recommend import _Users, pool_operands
    with torch.no_grad():
        users, dnn = pool_operands(model, _Users(np.zeros(len(history), np.int64), history, np.zeros(len(history), np.int64)),
                                   matrix, E.new_flag(matrix.device))
    A = users if users.dim() == 3 else users.unsqueeze(1)
    return AR.exact_and_bound(A, matrix[:pad], dnn, DEV)


@pytest.mark.parametrize("name", ["HiFiArk", "DKN"])
def test_recommend_matches_a_host_recompute(name, tmp_path):
    from newsrec_b200.recommend import recommend
    d = str(tmp_path)
    TE._write_validation_dir(d)
    u2i = os.path.join(d, "user2int.tsv")
    model = _model(name)
    k = 20
    files = {}
    for chunk in (1, 10 ** 9):
        files[chunk] = str(tmp_path / f"rec_{chunk}.tsv")
        n_lines = recommend(model, d, files[chunk], k, user2int_path=u2i, chunk_users=chunk)
    assert open(files[1], "rb").read() == open(files[10 ** 9], "rb").read()
    lines = _read(files[1])
    assert len(lines) == n_lines
    users, history, pad, ids, S, matrix = _host_scores(model, d, u2i)
    assert [u for u, _ in lines] == users
    _, E = _bound(model, matrix, history, pad)
    tol = 2 * E + 1e-6 * S.abs()  # the host recompute is itself fp32
    for u, (_, got) in enumerate(lines):
        hist = set(int(r) for r in history[u] if r != pad)
        rows = [ids.index(x) for x in got]
        assert not hist & set(rows)
        elig = [r for r in range(pad) if r not in hist]
        assert len(rows) == min(k, len(elig))
        kth = torch.sort(S[u, elig], descending=True).values[len(rows) - 1] if len(elig) >= k else float("-inf")
        for r in rows:
            assert S[u, r] >= kth - tol[u, r]
        for j in range(len(rows) - 1):
            assert S[u, rows[j]] >= S[u, rows[j + 1]] - tol[u, rows[j]] - tol[u, rows[j + 1]]
    # a category cap and MMR work through the file
    capped = str(tmp_path / "capped.tsv")
    recommend(model, d, capped, 10, user2int_path=u2i, max_per_category=1)
    from newsrec_b200 import evaluate as EV
    cat = dict(zip(ids, EV.read_news(d, ["category"])[1]["category"].tolist()))
    for _, got in _read(capped):
        assert len(set(cat[x] for x in got)) == len(got)
    mmr1, plain = str(tmp_path / "mmr1.tsv"), str(tmp_path / "plain.tsv")
    recommend(model, d, plain, 10, user2int_path=u2i)
    recommend(model, d, mmr1, 10, user2int_path=u2i, mmr_lambda=1.0)
    assert open(mmr1, "rb").read() == open(plain, "rb").read()
    recommend(model, d, str(tmp_path / "mmr.tsv"), 10, user2int_path=u2i, mmr_lambda=0.5)
