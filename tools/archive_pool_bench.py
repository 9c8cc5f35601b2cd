"""The --scorer hifiark / dkn arms of tools/recommend_bench.py and tools/pool_rank_bench.py: nr_topk_archive and
nr_pool_ranks_archive under the archive DNN click score, on seeded synthetic operands at the families' default shapes
(Hi-Fi Ark: P = 5 archive rows of F = 300, hidden 24; DKN: one user vector of F = 150, hidden 17).

Arms, each timed with CUDA events after a warm-up (median and best over reps):
  kernel       the library call over every user (its X / Y projections, planes, the pool kernel and the split merge);
  torch        a chunked torch restatement in fp32 (TF32 off): logits by matmul, softmax, the mix, relu, the output layer,
               then torch.topk (or the count of greater scores), timed on the first --baseline-users users;
  per-user     what a user can do without the pool kernels: nr_archive_score_fwd with the whole pool as every sampled user's
               candidates, then torch.topk, timed on the first --sample-users users.
Sample arms report their time and the time scaled to every user (linear in users: every user is scored alone).  Check: on
64 users, every returned score within the bound include/newsrec_b200.h states against fp64 (tests/archive_pool_ref.py).
"""
from __future__ import annotations

import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

SCORERS = {"hifiark": (5, 300, 24), "dkn": (1, 150, 17)}  # (P, F, hidden)


def add_args(ap):
    ap.add_argument("--scorer", choices=["dot"] + sorted(SCORERS), default="dot",
                    help="dot: users . news (the default arms); hifiark / dkn: the archive DNN click score at its default shape")
    ap.add_argument("--baseline-users", type=int, default=8192, help="users of the torch restatement arm (--scorer != dot)")
    ap.add_argument("--sample-users", type=int, default=256, help="users of the per-user nr_archive_score_fwd arm (--scorer != dot)")


def operands(scorer, U, n, dev, seed):
    import torch
    P, F, hid = SCORERS[scorer]
    g = torch.Generator(device=dev).manual_seed(seed)
    A = torch.randn(U, P, F, device=dev, generator=g)
    C = torch.randn(n, F, device=dev, generator=g)
    W1 = torch.randn(hid, 2 * F, device=dev, generator=g) / (2 * F) ** 0.5
    b1 = 0.1 * torch.randn(hid, device=dev, generator=g)
    w2 = torch.randn(1, hid, device=dev, generator=g) / hid ** 0.5
    b2 = 0.1 * torch.randn(1, device=dev, generator=g)
    return A, C, (W1, b1, w2, b2)


def torch_scores(A, C, dnn):
    """(u, n) fp32 scores of users A (u, P, F) against the pool C: the restatement of the score."""
    import torch
    W1, b1, w2, b2 = dnn
    F = C.shape[1]
    X = C @ W1[:, :F].T + b1                               # (n, hid)
    Y = A @ W1[:, F:].T                                    # (u, P, hid)
    w = torch.softmax(torch.einsum("upf,nf->unp", A, C), -1)
    return torch.relu(X[None] + torch.einsum("unp,uph->unh", w, Y)) @ w2.reshape(-1) + b2


def timed(fn, reps):
    import torch
    out, ts = None, []
    fn()
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return sorted(ts)[len(ts) // 2], min(ts), out


def _chunk(P, n):
    return max(1, (1 << 30) // (n * max(P, 32) * 4 * 3))


def _per_user(A, C, dnn, k, dev):
    import torch
    from newsrec_b200.ops_hifiark import score_impressions
    S, n, F = A.shape[0], C.shape[0], C.shape[1]
    if F % 4:  # the impression scorer takes rows of a multiple of 4 columns: zero columns, as DKN's own path widens them
        pad = lambda t: torch.nn.functional.pad(t, (0, 4 - F % 4))  # noqa: E731
        A, C, dnn = pad(A), pad(C), (torch.cat([pad(dnn[0][:, :F]), pad(dnn[0][:, F:])], 1),) + tuple(dnn[1:])
    cand = torch.arange(n, device=dev).repeat(S)
    seg = torch.arange(0, S * n + 1, n, device=dev)
    flag = torch.zeros(1, dtype=torch.int32, device=dev)
    return torch.topk(score_impressions(C, cand, seg, A, *dnn, flag).view(S, n), k, dim=1)


def recommend_arms(a, card):
    """tools/recommend_bench.py --scorer hifiark|dkn"""
    import json
    import torch
    import archive_pool_ref as AR
    from newsrec_b200 import require_cuda
    from newsrec_b200.ops import top_k_scores
    dev = require_cuda()
    torch.backends.cuda.matmul.allow_tf32 = False
    A, C, dnn = operands(a.scorer, a.users, a.news, dev, a.seed)
    P = A.shape[1]
    users = A[:, 0] if P == 1 else A
    cats = torch.randint(0, a.categories, (a.news,), device=dev, generator=torch.Generator(device=dev).manual_seed(a.seed + 1))
    m = a.max_per_category or 2
    Ub, Us = min(a.baseline_users, a.users), min(a.sample_users, a.users)
    results = []
    for k in a.k:
        r = dict(k=k)
        r["kernel_ms_median"], r["kernel_ms_best"], (ki, ks) = timed(lambda: top_k_scores(users, C, k, dnn=dnn), a.reps)
        r["capped_ms_median"], r["capped_ms_best"], (ci, _) = timed(
            lambda: top_k_scores(users, C, k, dnn=dnn, categories=cats, max_per_category=m), a.reps)
        ch = _chunk(P, a.news)

        def restated():
            outs = [torch.topk(torch_scores(A[lo:lo + ch], C, dnn), k, dim=1) for lo in range(0, Ub, ch)]
            return torch.cat([o.indices for o in outs])
        r["torch_ms_median"], r["torch_ms_best"], bi = timed(restated, a.reps)
        r["torch_users"] = Ub
        r["torch_ms_scaled_to_all_users"] = r["torch_ms_median"] * a.users / Ub
        r["per_user_ms_median"], r["per_user_ms_best"], _ = timed(
            lambda: [_per_user(A[lo:lo + 16], C, dnn, k, dev) for lo in range(0, Us, 16)], a.reps)
        r["per_user_users"] = Us
        r["per_user_ms_scaled_to_all_users"] = r["per_user_ms_median"] * a.users / Us
        rows = torch.linspace(0, a.users - 1, 64, device=dev).long()
        S, E = AR.exact_and_bound(A[rows], C, dnn, dev)
        s_k, e_k = torch.gather(S, 1, ki[rows]), torch.gather(E, 1, ki[rows])
        r["scores_within_bound"] = bool(((ks[rows].double() - s_k).abs() <= e_k).all())
        kth = torch.topk(S, k, dim=1).values[:, -1:]
        r["set_within_bound"] = bool((s_k >= kth - 2 * e_k).all())
        sample = rows[rows < Ub]
        r["same_set_as_torch_share"] = float((torch.sort(ki[sample], 1).values == torch.sort(bi[sample], 1).values).all(1).float().mean())
        r["capped_max_per_category"] = int(max(torch.bincount(cats[ci[u][ci[u] >= 0]]).max() for u in rows.tolist()))
        print(f"k={k}: nr_topk_archive {r['kernel_ms_median']:.1f} ms, capped (m={m}) {r['capped_ms_median']:.1f} ms; "
              f"torch restatement {r['torch_ms_median']:.1f} ms for {Ub} users ({r['torch_ms_scaled_to_all_users']:.0f} ms scaled); "
              f"per-user nr_archive_score_fwd + topk {r['per_user_ms_median']:.1f} ms for {Us} users "
              f"({r['per_user_ms_scaled_to_all_users']:.0f} ms scaled); checks {r['scores_within_bound'] and r['set_within_bound']}",
              flush=True)
        results.append(r)
    Pn, F, hid = SCORERS[a.scorer]
    print(json.dumps(dict(card=card(), scorer=a.scorer, P=Pn, F=F, hidden=hid, users=a.users, news=a.news, reps=a.reps,
                          max_per_category=m, categories=a.categories, results=results)))
    return 0


def rank_arms(a, card):
    """tools/pool_rank_bench.py --scorer hifiark|dkn: one or two targets per row and 0 to 50 exclusions, as the dot arms"""
    import json
    import torch
    import archive_pool_ref as AR
    from newsrec_b200 import require_cuda
    from newsrec_b200.ops import pool_ranks, top_k_scores
    dev = require_cuda()
    torch.backends.cuda.matmul.allow_tf32 = False
    Q, n = a.rows, a.news
    A, C, dnn = operands(a.scorer, Q, n, dev, a.seed)
    P = A.shape[1]
    users = A[:, 0] if P == 1 else A
    g = torch.Generator(device=dev).manual_seed(a.seed + 2)
    n_t = 1 + (torch.rand(Q, device=dev, generator=g) < 0.5).long()
    t_off = torch.zeros(Q + 1, dtype=torch.int64, device=dev)
    t_off[1:] = torch.cumsum(n_t, 0)
    t_row = torch.randint(0, n, (int(t_off[-1]),), device=dev, generator=g)
    second = torch.arange(len(t_row), device=dev) == t_off[:-1].repeat_interleave(n_t) + 1  # a row's two targets differ
    t_row[second] = (t_row[second.roll(-1)] + 1 + torch.randint(0, n - 1, (int(second.sum()),), device=dev, generator=g)) % n
    n_x = torch.randint(0, 51, (Q,), device=dev, generator=g)
    x_off = torch.zeros(Q + 1, dtype=torch.int64, device=dev)
    x_off[1:] = torch.cumsum(n_x, 0)
    x_row = torch.randint(0, n, (int(x_off[-1]),), device=dev, generator=g)
    r = dict(card=card(), scorer=a.scorer, rows=Q, news=n, targets=len(t_row), reps=a.reps)
    r["pool_ranks_ms_median"], r["pool_ranks_ms_best"], (rank, score) = timed(
        lambda: pool_ranks(users, C, t_row, t_off, x_row, x_off, dnn=dnn), a.reps)
    r["topk10_ms_median"], r["topk10_ms_best"], _ = timed(lambda: top_k_scores(users, C, 10, x_row, x_off, dnn=dnn), a.reps)
    Ub = min(a.baseline_users, Q)
    ch = _chunk(P, n)
    t_q = torch.arange(Q, device=dev).repeat_interleave(n_t)
    x_q = torch.arange(Q, device=dev).repeat_interleave(n_x)

    def restated():
        out = []
        cols = torch.arange(n, device=dev)
        for lo in range(0, Ub, ch):
            hi = min(Ub, lo + ch)
            S = torch_scores(A[lo:hi], C, dnn)
            ta, tb, xa, xb = int(t_off[lo]), int(t_off[hi]), int(x_off[lo]), int(x_off[hi])
            qt, rt = t_q[ta:tb] - lo, t_row[ta:tb]
            st = S[qt, rt]
            S[x_q[xa:xb] - lo, x_row[xa:xb]] = float("nan")
            S[qt, rt] = float("nan")
            Sq = S[qt]
            out.append(((Sq > st[:, None]) | ((Sq == st[:, None]) & (cols[None, :] < rt[:, None]))).sum(1))
        return torch.cat(out)
    r["torch_ms_median"], r["torch_ms_best"], base = timed(restated, a.reps)
    r["torch_rows"] = Ub
    r["torch_ms_scaled_to_all_rows"] = r["torch_ms_median"] * Q / Ub
    nt = len(base)
    r["ranks_equal_to_torch_share"] = float((rank[:nt] == base).double().mean())
    inband = checked = 0
    for q in torch.linspace(0, Q - 1, 32).long().tolist():
        S, E = AR.exact_and_bound(A[q:q + 1], C, dnn, dev)
        S, E = S[0], E[0]
        elig = torch.ones(n, dtype=torch.bool, device=dev)
        elig[x_row[int(x_off[q]):int(x_off[q + 1])]] = False
        ts = t_row[int(t_off[q]):int(t_off[q + 1])]
        elig[ts] = False
        for j, t in enumerate(ts.tolist()):
            d, e = S - S[t], E + E[t]
            inband += int((elig & (d > e)).sum()) <= int(rank[int(t_off[q]) + j]) <= int((elig & (d >= -e)).sum())
            checked += 1
    r["checked_targets"], r["kernel_in_band"] = checked, inband
    print(f"nr_pool_ranks_archive {r['pool_ranks_ms_median']:.1f} ms, nr_topk_archive k=10 {r['topk10_ms_median']:.1f} ms, "
          f"torch restatement {r['torch_ms_median']:.1f} ms for {Ub} rows ({r['torch_ms_scaled_to_all_rows']:.0f} ms scaled); "
          f"band {inband}/{checked}", flush=True)
    print(json.dumps(r))
    return 0

