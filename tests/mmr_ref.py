"""fp64 restatement of nr_mmr_rerank (include/newsrec_b200.h) and a path verifier for the kernel's output.

The contract, for user u with shortlist entries (rows r_i, score bits s_i) before the first -1:
    rel_i = (s_i - s_min) / (s_max - s_min)  (1 for all when s_max == s_min)
    sim(i, j) = cosine of the news rows r_i and r_j, 0 when either is all zeros
    greedy: min(k, live) times, take the i not yet taken with the largest
            obj_i = lam rel_i - (1 - lam) max_{j taken} sim(i, j)   (0 while nothing is taken),
            equal objectives to the lower position.
``mmr_fp64`` runs the greedy in fp64.  ``verify_path`` follows the kernel's own picks instead: given its earlier picks, each
pick's fp64 objective must be within 2 e_obj of the best remaining one, with e_obj the header's bound.  That is robust to
near-ties, which the fp32 kernel may break either way."""
import numpy as np


def eps(D):
    """The hi/lo tensor-core dot product bound factor of nr_topk_dot: 2^-15 + 3 round_up(D, 64) 2^-23."""
    return 2.0 ** -15 + 3 * (-(-D // 64) * 64) * 2.0 ** -23


def e_sim(D):
    """Bound between the kernel's similarity and the exact cosine of the fp32 rows: c eps + 2^-21, c = 2 / (1 - eps)."""
    e = eps(D)
    return 2 * e / (1 - e) + 2.0 ** -21


def e_obj(D, lam):
    """Bound between the kernel's objective and fp64 on the same score bits and the fp32 lam: (1 - lam) e_sim + 2^-20."""
    lam = float(np.float32(lam))
    return (1 - lam) * e_sim(D) + 2.0 ** -20


def _live(sl_idx):
    """Number of entries before the first -1 of each row of sl_idx (U, L)."""
    dead = np.asarray(sl_idx) == -1
    return np.where(dead.any(1), dead.argmax(1), dead.shape[1])


def _user_terms(news, rows, scores):
    """(rel (L,), cos (L, L)) in fp64 of one user's live entries."""
    s = np.asarray(scores, np.float32).astype(np.float64)
    smax, smin = s.max(), s.min()
    rel = np.ones_like(s) if smax == smin else (s - smin) / (smax - smin)
    X = np.asarray(news, np.float32).astype(np.float64)[np.asarray(rows, np.int64)]
    nrm = np.linalg.norm(X, axis=1)
    Xn = np.divide(X, nrm[:, None], out=np.zeros_like(X), where=nrm[:, None] > 0)
    return rel, Xn @ Xn.T


def _objective(rel, cos, taken, lam):
    lam = float(np.float32(lam))
    msim = cos[:, taken].max(1) if taken else np.zeros(len(rel))
    return lam * rel - (1 - lam) * msim


def mmr_fp64(news, sl_idx, sl_score, k, lam):
    """The contract's greedy in fp64: (idx (U, k) int64, score (U, k) fp32), -1 / -inf after the last pick."""
    sl_idx, sl_score = np.asarray(sl_idx, np.int64), np.asarray(sl_score, np.float32)
    U = sl_idx.shape[0]
    idx = np.full((U, k), -1, np.int64)
    sc = np.full((U, k), -np.inf, np.float32)
    for u, L in enumerate(_live(sl_idx)):
        if L == 0:
            continue
        rel, cos = _user_terms(news, sl_idx[u, :L], sl_score[u, :L])
        taken = []
        for t in range(min(k, L)):
            obj = _objective(rel, cos, taken, lam)
            obj[taken] = -np.inf
            i = int(np.argmax(obj))  # the first maximum: equal objectives go to the lower position
            taken.append(i)
            idx[u, t], sc[u, t] = sl_idx[u, i], sl_score[u, i]
    return idx, sc


def verify_path(news, sl_idx, sl_score, idx, score, k, lam):
    """Asserts that (idx, score) is a valid output of nr_mmr_rerank for the shortlist (sl_idx, sl_score) over the pool news
    (n, D): min(k, live) distinct picks from the live entries, each with the shortlist's own score bits, then -1 / -inf; and
    at every step the pick's fp64 objective, given the kernel's earlier picks, within 2 e_obj of the best remaining one."""
    news = np.asarray(news, np.float32)
    sl_idx, sl_score = np.asarray(sl_idx, np.int64), np.asarray(sl_score, np.float32)
    idx, score = np.asarray(idx, np.int64), np.asarray(score, np.float32)
    assert idx.shape == score.shape == (sl_idx.shape[0], k), (idx.shape, score.shape)
    tol = 2 * e_obj(news.shape[1], lam)
    for u, L in enumerate(_live(sl_idx)):
        n_pick = min(k, L)
        assert (idx[u, n_pick:] == -1).all() and (score[u, n_pick:] == -np.inf).all(), (u, idx[u], score[u])
        if n_pick == 0:
            continue
        pos_of = {int(r): i for i, r in reversed(list(enumerate(sl_idx[u, :L])))}
        rel, cos = _user_terms(news, sl_idx[u, :L], sl_score[u, :L])
        taken = []
        for t in range(n_pick):
            r = int(idx[u, t])
            assert r in pos_of, (u, t, r, "not a live shortlist row")
            # duplicated rows in a shortlist do not come from nr_topk_dot; take the first position not yet taken
            cands = [i for i in range(L) if sl_idx[u, i] == r and i not in taken]
            assert cands, (u, t, r, "picked twice")
            i = cands[0]
            assert score[u, t].view(np.int32) == sl_score[u, i].view(np.int32), (u, t, score[u, t], sl_score[u, i])
            obj = _objective(rel, cos, taken, lam)
            rest = np.ones(L, bool)
            rest[taken] = False
            best = obj[rest].max()
            assert obj[i] >= best - tol, (u, t, i, obj[i], best, tol)
            taken.append(i)
