"""Windowed against whole-pool top-k and ranks on the GPU: nr_topk_dot and nr_pool_ranks over every news, against their
_ranged variants over each request's 48-hour window of the same pool (newsrec_b200.window), at recommend's shape.

Shape: 700k users x 120k news, D = 300 (seeded synthetic fp32 vectors).  Every news gets a first-shown time uniform over 42
days and the pool is in that time order; request times are uniform over the same 42 days and the users are sorted by them,
as recommend and pool_eval sort each chunk; W = 48 h, so a window holds about 1/21 of the pool.  Ranks: one target per row,
drawn from its window.

    python tools/pool_window_bench.py [--users 700000] [--news 120000] [--dim 300] [--hours 48] [--days 42] [--reps 3]

Time: CUDA events around ops.top_k_scores (k = 10 and k = 100) and ops.pool_ranks (operand planes, kernel, split merge and
the flag read-back), after a warm-up, the arms alternating within each repetition; medians and minima over reps.  Checks,
bit for bit: on a few sampled rows, the ranged lists against the unranged call with every news outside the row's window
excluded (a few rows only: the kernels scan a row's exclusion list linearly, and a complement holds ~95 % of the pool); on
more sampled rows, the ranged lists and ranks against the unranged calls on the row's window alone (rows shifted back).
Prints the card name and power limit, a line per repetition, then one JSON line.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "news-recommendation_b200", "src"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from recommend_bench import card  # noqa: E402


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--users", type=int, default=700_000)
    ap.add_argument("--news", type=int, default=120_000)
    ap.add_argument("--dim", type=int, default=300)
    ap.add_argument("--hours", type=float, default=48.0)
    ap.add_argument("--days", type=float, default=42.0)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sample", type=int, default=128, help="rows checked against the unranged call on their window")
    ap.add_argument("--sample-excluded", type=int, default=8, help="rows checked against the complement-excluded call")
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args(argv)
    import numpy as np
    import torch
    from newsrec_b200 import require_cuda
    from newsrec_b200.ops import pool_ranks, top_k_scores
    from newsrec_b200.window import PoolWindow
    print(f"card: {card()}", flush=True)
    dev = require_cuda()
    g = torch.Generator(device=dev).manual_seed(a.seed)
    U, n, D = a.users, a.news, a.dim
    users = torch.randn(U, D, device=dev, generator=g)
    news = torch.randn(n, D, device=dev, generator=g)
    rng = np.random.default_rng(a.seed)
    span = int(a.days * 86400)
    pw = PoolWindow(np.sort(rng.integers(0, span, n)), np.ones(n, bool))  # the pool in time order already
    t_req = np.sort(rng.integers(0, span, U))
    lo, hi = pw.ranges(t_req, a.hours * 3600.0)
    rr = (torch.from_numpy(lo).to(dev), torch.from_numpy(hi).to(dev))
    live = hi > lo
    tgt = torch.from_numpy(np.where(live, lo + (rng.random(U) * np.maximum(hi - lo, 1)).astype(np.int64), 0))
    t_off = torch.arange(U + 1, dtype=torch.int64)
    arms = {
        "topk10_pool": lambda: top_k_scores(users, news, 10),
        "topk10_window": lambda: top_k_scores(users, news, 10, row_range=rr),
        "topk100_pool": lambda: top_k_scores(users, news, 100),
        "topk100_window": lambda: top_k_scores(users, news, 100, row_range=rr),
        "ranks_pool": lambda: pool_ranks(users, news, tgt, t_off),
        "ranks_window": lambda: pool_ranks(users, news, tgt, t_off, row_range=rr),
    }
    for f in arms.values():
        f()
    torch.cuda.synchronize()
    ms = {name: [] for name in arms}
    for rep in range(a.reps):
        for name, f in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            f()
            e1.record()
            e1.synchronize()
            ms[name].append(e0.elapsed_time(e1))
        print(f"rep {rep}: " + ", ".join(f"{k} {v[-1]:.1f} ms" for k, v in ms.items()), flush=True)

    def same(x, y):
        return bool(torch.equal(x[0], y[0]) and torch.equal(x[1].view(torch.int32), y[1].view(torch.int32)))

    def sample(size):
        s = np.sort(rng.choice(np.flatnonzero(live), size=min(size, int(live.sum())), replace=False))
        sd = torch.from_numpy(s).to(dev)
        return s, users[sd], (rr[0][sd], rr[1][sd])

    equal = {}
    s, su, srr = sample(a.sample_excluded)  # against the complement excluded
    comp = [np.concatenate([np.arange(0, lo[i]), np.arange(hi[i], n)]) for i in s]
    xo = torch.from_numpy(np.concatenate([[0], np.cumsum([len(c) for c in comp])]).astype(np.int64))
    xr = torch.from_numpy(np.concatenate(comp).astype(np.int64))
    equal["topk_vs_excluded"] = all(same(top_k_scores(su, news, k, row_range=srr), top_k_scores(su, news, k, xr, xo))
                                    for k in (10, 100))
    s, su, srr = sample(a.sample)  # against the unranged calls on each row's window
    ok = True
    for j, i in enumerate(s):
        part = news[int(lo[i]):int(hi[i])]
        for k in (10, 100):
            got = top_k_scores(su[j:j + 1], news, k, row_range=(srr[0][j:j + 1], srr[1][j:j + 1]))
            idx, sc = top_k_scores(su[j:j + 1], part, k)
            ok &= same(got, (torch.where(idx >= 0, idx + int(lo[i]), idx), sc))
        got = pool_ranks(su[j:j + 1], news, tgt[i:i + 1], torch.arange(2), row_range=(srr[0][j:j + 1], srr[1][j:j + 1]))
        ok &= same(got, pool_ranks(su[j:j + 1], part, tgt[i:i + 1] - int(lo[i]), torch.arange(2)))
    equal["topk_and_ranks_vs_window_alone"] = ok
    tiles_pool = (n + 63) // 64
    blk_lo, blk_hi = lo.reshape(-1)[:U // 64 * 64].reshape(-1, 64), hi[:U // 64 * 64].reshape(-1, 64)
    tiles_window = float(np.mean((blk_hi.max(1) + 63) // 64 - blk_lo.min(1) // 64))
    out = {"card": card(), "users": U, "news": n, "dim": D, "hours": a.hours, "days": a.days, "reps": a.reps,
           "window_mean": float(np.mean(hi - lo)), "tiles_per_block_pool": tiles_pool,
           "tiles_per_block_window_mean": tiles_window, "sample_rows": [a.sample_excluded, a.sample], "bit_equal": equal}
    for name, v in ms.items():
        out[f"{name}_ms_median"] = round(statistics.median(v), 2)
        out[f"{name}_ms_min"] = round(min(v), 2)
    print(json.dumps(out))
    return 0 if all(equal.values()) else 1


if __name__ == "__main__":
    sys.exit(main())
