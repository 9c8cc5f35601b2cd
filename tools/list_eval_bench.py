"""nr_list_stats on the GPU at MIND-large's shape: the pair-similarity sums and distinct-category counts of --lists lists of k
news (the statistics behind pool_eval.evaluate_lists' ils@K and distinct_<field>@K) over a clustered pool of --news x --dim
fp32 news vectors (--stories centroids plus noise, as tools/recommend_bench.py --mmr-lambda builds it; a news' category is its
story).  The lists are uniform random rows of the pool, so the row gathers see little cache reuse.

Two arms alternate in the same run at every k: the kernel (one raw nr_list_stats call, cut-offs (1, 5, k) or fewer) and a
torch restatement of it (in chunks of --baseline-chunk lists: gather, row norms, bmm Gram in fp32 with TF32 off, the
strictly lower triangle summed in fp64 per row and prefix-summed over the rows, distinct categories of the sorted prefixes).
Time: CUDA events around each arm after a warm-up, median and best over --reps.  Checks: --sample lists against the exact
fp64 cosines of the fp32 rows, each pair sum within the header's bound (pairs x e_sim + pairs^2 2^-52); the distinct counts
of every list equal the restatement's.  Prints the card name and power limit, then one JSON line.

    python tools/list_eval_bench.py [--lists 700000] [--news 120000] [--dim 300] [--k 10 100 128] [--stories 2000]
                                    [--reps 5] [--baseline-chunk 8192] [--sample 256] [--seed 0]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "news-recommendation_b200", "src"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from recommend_bench import card  # noqa: E402


def e_sim(D):
    """nr_mmr_rerank's / nr_list_stats' similarity bound (include/newsrec_b200.h)."""
    eps = 2.0 ** -15 + 3 * (-(-D // 64) * 64) * 2.0 ** -23
    return 2 * eps / (1 - eps) + 2.0 ** -21


def torch_list_stats(news, cats, idx, ks, chunk):
    """The restatement: (pair_sum (R, n_ks) fp64, distinct (R, n_ks) int32) of full lists idx (R, k)."""
    import torch
    out_p, out_d = [], []
    for lo in range(0, idx.shape[0], chunk):
        rows = idx[lo:lo + chunk]
        X = news[rows]                                                    # (c, k, D) fp32
        nrm = X.norm(dim=2, keepdim=True)
        Xn = torch.where(nrm > 0, X / nrm, torch.zeros_like(X))
        G = torch.bmm(Xn, Xn.transpose(1, 2))
        pref = torch.tril(G, diagonal=-1).double().sum(2).cumsum(1)      # sum_{j < K} sum_{i < j}
        out_p.append(torch.stack([pref[:, K - 1] for K in ks], 1))
        c = cats[rows]
        d = []
        for K in ks:
            s = torch.sort(c[:, :K], 1).values
            d.append(1 + (s[:, 1:] != s[:, :-1]).sum(1).int())
        out_d.append(torch.stack(d, 1))
    return torch.cat(out_p), torch.cat(out_d)


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--lists", type=int, default=700_000)
    ap.add_argument("--news", type=int, default=120_000)
    ap.add_argument("--dim", type=int, default=300)
    ap.add_argument("--k", type=int, nargs="+", default=[10, 100, 128])
    ap.add_argument("--stories", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--baseline-chunk", type=int, default=8192, help="lists per torch pass")
    ap.add_argument("--sample", type=int, default=256, help="lists checked against fp64")
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args(argv)
    if not all(1 <= k <= 128 for k in a.k) or a.lists < 1 or a.news < 1 or not 1 <= a.dim <= 4096:
        ap.error("--k in [1, 128]; --lists, --news at least 1; --dim in [1, 4096]")
    import numpy as np
    import torch
    from newsrec_b200 import check, load_library, require_cuda
    from newsrec_b200.ops import _p, _stream
    dev = require_cuda()
    lib = load_library()
    torch.backends.cuda.matmul.allow_tf32 = False
    g = torch.Generator(device=dev).manual_seed(a.seed)
    story = torch.randint(0, a.stories, (a.news,), device=dev, generator=g)
    centroids = torch.randn(a.stories, a.dim, device=dev, generator=g)
    news = (centroids[story] + 0.3 * torch.randn(a.news, a.dim, device=dev, generator=g)).contiguous()
    cats = story.int().contiguous()
    print(f"card: {card()}", flush=True)
    results = []
    for k in a.k:
        ks = tuple(sorted({x for x in (1, 5) if x < k} | {k}))
        idx = torch.randint(0, a.news, (a.lists, k), device=dev, generator=g)
        pair_sum = torch.empty((a.lists, len(ks)), dtype=torch.float64, device=dev)
        distinct = torch.empty((a.lists, len(ks)), dtype=torch.int32, device=dev)
        flag = torch.zeros(1, dtype=torch.int32, device=dev)
        c_ks = (C.c_int * len(ks))(*ks)

        def kernel():
            check(lib.nr_list_stats(_p(news), a.news, a.dim, a.dim, _p(idx), a.lists, k, _p(cats), c_ks, len(ks), _p(pair_sum),
                                    _p(distinct), _p(flag), _stream()), "nr_list_stats")

        def baseline():
            return torch_list_stats(news, cats, idx, ks, a.baseline_chunk)

        def timed(fn):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            out = fn()
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1), out

        kernel(), baseline()  # warm-up
        tk, tb = [], []
        for _ in range(a.reps):
            tk.append(timed(kernel)[0])
            t, (bp, bd) = timed(baseline)
            tb.append(t)
        assert int(flag.item()) == 0
        # checks: sampled lists against the exact cosines, the distinct counts against the restatement
        rows = torch.linspace(0, a.lists - 1, min(a.sample, a.lists), device=dev).long()
        X = news.double()
        Xn = X / X.norm(dim=1, keepdim=True)
        S = Xn[idx[rows]]
        exact = torch.tril(torch.bmm(S, S.transpose(1, 2)), diagonal=-1).sum(2).cumsum(1)
        pairs = torch.tensor([K * (K - 1) / 2 for K in ks], dtype=torch.float64, device=dev)
        want = torch.stack([exact[:, K - 1] for K in ks], 1)
        bound = pairs * e_sim(a.dim) + pairs ** 2 * 2.0 ** -52
        err = (pair_sum[rows] - want).abs()
        worst = float((err / bound.clamp_min(1e-300)).max())
        assert worst <= 1.0, worst
        assert torch.equal(distinct, bd)
        per_pair = pairs.clamp_min(1)
        res = dict(k=k, ks=list(ks), kernel_ms_median=statistics.median(tk), kernel_ms_best=min(tk),
                   torch_ms_median=statistics.median(tb), torch_ms_best=min(tb),
                   speedup_median=statistics.median(tb) / statistics.median(tk),
                   worst_error_over_bound=worst, max_error_per_pair=float((err / per_pair).max()),
                   max_kernel_vs_torch_per_pair=float(((pair_sum - bp).abs() / per_pair).max()),
                   mean_ils_at_k=float((pair_sum[:, -1] / pairs[-1].clamp_min(1)).mean()) if k >= 2 else float("nan"),
                   distinct_equal=True)
        print(f"k={k}: nr_list_stats {res['kernel_ms_median']:.2f} ms, torch {res['torch_ms_median']:.1f} ms "
              f"(x{res['speedup_median']:.1f}); error / bound {worst:.3g}", flush=True)
        results.append(res)
        del idx, pair_sum, distinct, bp, bd
        torch.cuda.empty_cache()
    print(json.dumps(dict(card=card(), lists=a.lists, news=a.news, dim=a.dim, stories=a.stories, reps=a.reps,
                          baseline_chunk=a.baseline_chunk, results=results), default=float))
    return 0


if __name__ == "__main__":
    sys.exit(main())
