"""MMR re-ranking on the H100: nr_mmr_rerank / ops.top_k_scores(..., mmr_lambda=, mmr_depth=) and
newsrec_b200.recommend(..., mmr_lambda=, mmr_depth=), checked against the contract of include/newsrec_b200.h.

The shortlist is nr_topk_dot's top depth (ops.top_k_scores at k = depth, deterministic, so the same list the re-ranking
starts from).  tests/mmr_ref.verify_path follows the kernel's picks: each must be a live shortlist entry with the shortlist's
own score bits, and its fp64 objective, given the kernel's earlier picks, within 2 e_obj of the best remaining one (e_obj the
header's bound).  The exact cases (lambda = 1, depth == k, repeated calls) are compared bit for bit."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import mmr_ref as M
import test_gpu_evaluate as TE
import test_gpu_recommend as TR

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
LAMBDAS = (0.0, 0.25, 0.5, 0.9, 1.0)


def _pool(kind, n, D, seed):
    g = torch.Generator().manual_seed(seed)
    if kind == "random":
        return torch.randn(n, D, generator=g)
    stories = torch.randn(20, D, generator=g)  # story centroids plus noise
    return stories[torch.randint(0, 20, (n,), generator=g)] + 0.15 * torch.randn(n, D, generator=g)


def _run(users, news, k, lam, depth, excl=(None, None)):
    from newsrec_b200.ops import top_k_scores
    sl_idx, sl_score = top_k_scores(users, news, depth, *excl)
    idx, score = top_k_scores(users, news, k, *excl, mmr_lambda=lam, mmr_depth=depth)
    return sl_idx, sl_score, idx, score


def _verify(news, sl_idx, sl_score, idx, score, k, lam):
    M.verify_path(news.cpu().numpy(), sl_idx.cpu().numpy(), sl_score.cpu().numpy(), idx.cpu().numpy(), score.cpu().numpy(),
                  k, lam)


@pytest.mark.parametrize("depth", [1, 37, 64, 65, 128])
@pytest.mark.parametrize("D", [1, 8, 63, 64, 300, 400, 1000])
def test_path_verifier_over_the_grid(D, depth):
    from newsrec_b200.ops import top_k_scores
    for kind in ("random", "clustered"):
        news = _pool(kind, 300, D, seed=D * 1000 + depth)
        users = torch.randn(12, D, generator=torch.Generator().manual_seed(D + depth))
        for k in sorted({1, min(10, depth), depth}):
            for lam in LAMBDAS:
                sl_idx, sl_score, idx, score = _run(users, news, k, lam, depth)
                _verify(news, sl_idx, sl_score, idx, score, k, lam)
                if lam == 1.0:  # the plain k-list, bit for bit
                    pi, ps = top_k_scores(users, news, k)
                    assert torch.equal(idx, pi) and torch.equal(score, ps), (kind, k)
                if k == depth:  # the shortlist's set, reordered
                    assert torch.equal(torch.sort(idx, 1).values, torch.sort(sl_idx, 1).values), (kind, lam)


def test_fewer_eligible_news_than_depth_pad_the_output():
    n, D = 40, 24
    news = _pool("clustered", n, D, seed=3)
    users = torch.randn(4, D, generator=torch.Generator().manual_seed(4))
    excl = [list(range(35)), [], list(range(0, 40, 2)), list(range(40))]  # 5, 40, 20 and 0 eligible news
    rows, offs = TR._csr(excl)
    for k, depth in ((10, 64), (30, 30), (1, 128)):
        for lam in (0.0, 0.5, 1.0):
            sl_idx, sl_score, idx, score = _run(users, news, k, lam, depth, (rows, offs))
            assert [int((sl_idx[u] >= 0).sum()) for u in range(4)] == [min(depth, e) for e in (5, 40, 20, 0)]
            _verify(news, sl_idx, sl_score, idx, score, k, lam)
            live = (idx >= 0).sum(1).tolist()
            assert live == [min(k, depth, e) for e in (5, 40, 20, 0)], live
            assert bool((score[idx < 0] == float("-inf")).all())
            for u, lst in enumerate(excl):
                assert not set(idx[u].tolist()) & set(lst)


def test_planted_stories_come_out_distinct():
    # 20 stories x 5 near-duplicates: news (s, j) = e_s + 0.1 e_{20 + 5s + j}, row 5s + j.  A user scores story s at a
    # distinct w_s and every duplicate of a story alike; cosines are 1 / 1.01 within a story and 0 across stories.
    S, J, D = 20, 5, 20 + 100
    news = torch.zeros(S * J, D)
    for s in range(S):
        for j in range(J):
            news[J * s + j, s] = 1.0
            news[J * s + j, S + J * s + j] = 0.1
    g = torch.Generator().manual_seed(7)
    ranks = [torch.randperm(S, generator=g) for _ in range(6)]
    users = torch.zeros(6, D)
    for u, r in enumerate(ranks):
        users[u, :S] = 10.0 - 0.2 * r.float()  # story with rank 0 first
    from newsrec_b200.ops import top_k_scores
    plain, _ = top_k_scores(users, news, 10)
    mmr, _ = top_k_scores(users, news, 10, mmr_lambda=0.5, mmr_depth=100)
    for u, r in enumerate(ranks):
        order = torch.argsort(r).tolist()  # stories best first
        assert len({x // J for x in plain[u].tolist()}) == 2
        assert plain[u].tolist() == [J * order[0] + j for j in range(J)] + [J * order[1] + j for j in range(J)]
        assert mmr[u].tolist() == [J * s for s in order[:10]], (u, mmr[u].tolist())


def test_two_calls_give_the_same_bits():
    news = _pool("clustered", 5000, 300, seed=11)
    users = torch.randn(3000, 300, generator=torch.Generator().manual_seed(12))
    from newsrec_b200.ops import top_k_scores
    a = top_k_scores(users, news, 10, mmr_lambda=0.5, mmr_depth=128)
    b = top_k_scores(users, news, 10, mmr_lambda=0.5, mmr_depth=128)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1].view(torch.int32), b[1].view(torch.int32))
    sl = top_k_scores(users, news, 128)
    rows = torch.linspace(0, 2999, 40).long()
    _verify(news, sl[0][rows], sl[1][rows], a[0][rows], a[1][rows], 10, 0.5)


def test_a_shortlist_row_outside_the_pool_sets_the_flag():
    from newsrec_b200 import load_library
    from newsrec_b200.ops import _p, _stream
    lib = load_library()
    n, D, depth, k = 50, 16, 8, 4
    news = torch.randn(n, D, device=DEV)
    sl_score = torch.linspace(1, 0, depth, device=DEV).repeat(3, 1).contiguous()
    cases = [([0, 1, 2, 3, 4, 5, 6, 7], 0), ([0, 1, n, 3, 4, 5, 6, 7], 1), ([0, -5, 2, 3, 4, 5, 6, 7], 1),
             ([0, 1, 2, -1, n + 7, -9, 6, 7], 0)]  # entries after the first -1 are ignored
    for rows, want in cases:
        sl_idx = torch.tensor([rows, [1, 2, 3, 4, 5, 6, 7, 8], rows], dtype=torch.int64, device=DEV)
        idx = torch.empty((3, k), dtype=torch.int64, device=DEV)
        score = torch.empty((3, k), dtype=torch.float32, device=DEV)
        flag = torch.zeros(1, dtype=torch.int32, device=DEV)
        rc = lib.nr_mmr_rerank(_p(news), n, D, D, _p(sl_idx), _p(sl_score), 3, depth, k, 0.5, _p(idx), _p(score), _p(flag),
                               _stream())
        assert rc == 0, lib.nr_last_error().decode()
        assert int(flag.item()) == want, rows
        if want == 0:
            _verify(news, sl_idx, sl_score, idx, score, k, 0.5)


@pytest.mark.parametrize("name", ["NRMS", "NAML"])
def test_recommend_end_to_end(name, tmp_path):
    from newsrec_b200 import evaluate as E
    from newsrec_b200.ops import top_k_scores
    from newsrec_b200.recommend import _Users, exclusion_csr, recommend
    d = str(tmp_path)
    TE._write_validation_dir(d)
    u2i = os.path.join(d, "user2int.tsv")
    model = TR._model(name)
    k, depth, lam = 10, 40, 0.5
    files = {}
    for chunk, mmr in ((7, lam), (10 ** 9, lam), (10 ** 9, 1.0), (10 ** 9, None)):
        files[chunk, mmr] = str(tmp_path / f"rec_{chunk}_{mmr}.tsv")
        recommend(model, d, files[chunk, mmr], k, user2int_path=u2i, chunk_users=chunk, mmr_lambda=mmr,
                  mmr_depth=None if mmr is None else depth)
    data = {key: open(f, "rb").read() for key, f in files.items()}
    assert data[7, lam] == data[10 ** 9, lam]
    assert data[10 ** 9, 1.0] == data[10 ** 9, None]
    assert data[10 ** 9, lam] != data[10 ** 9, None]
    # the host restatement: recommend's user vectors and exclusions, the shortlist, the lines through the path verifier
    with torch.no_grad():
        index, matrix = E.news_matrix(model, d)
        pad = index["PADDED_NEWS"]
        user, history, length, _ = E.user_tables(E.read_behaviors(d), index, model.config.num_clicked_news_a_user, u2i)
        uv = E.user_vectors(model, _Users(user, history, length), matrix, E.new_flag(matrix.device))
    rows, offs = exclusion_csr(history, pad)
    pool = matrix[:pad]
    sl_idx, sl_score = top_k_scores(uv, pool, depth, torch.from_numpy(rows), torch.from_numpy(offs))
    ids = E.read_news(d, [])[0]
    lines = TR._read(files[10 ** 9, lam])
    assert len(lines) == uv.shape[0]
    sl_i, sl_s = sl_idx.cpu().numpy(), sl_score.cpu().numpy()
    idx = np.full((len(lines), k), -1, np.int64)
    score = np.full((len(lines), k), -np.inf, np.float32)
    for u, (_, got) in enumerate(lines):
        for t, x in enumerate(got):
            idx[u, t] = ids.index(x)
            score[u, t] = sl_s[u][list(sl_i[u]).index(idx[u, t])]
    M.verify_path(pool.cpu().numpy(), sl_i, sl_s, idx, score, k, lam)
