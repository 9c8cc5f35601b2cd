"""nr_topk_dot on the GPU at MIND-large's shape: the k best of n_news news for n_users users (seeded synthetic fp32 vectors,
D = 300 as NRMS's), against chunked torch.matmul in fp32 (TF32 off) + torch.topk over the same inputs, the two timed
alternately in the same run.  The baseline's answer also cross-checks the kernel's: every returned score within the bound of
include/newsrec_b200.h of the fp32 product, and the set equal up to news within twice the bound of the k-th best.

Diversified lists (--max-per-category M): every news gets a synthetic category, drawn from --categories N keys with
probability proportional to 1 / rank^s (--zipf s; 0 is uniform), and nr_topk_dot_capped is timed against the plain
nr_topk_dot at the same k, the two alternating in the same run (no matmul baseline).  The sampled users' capped lists are
checked: no category over M, scores within the bound, and with M >= k the plain lists bit for bit.

Diversified by content (--mmr-lambda X [--mmr-depth L]): the news are clustered (--stories centroids plus noise, as near-copies
of one story are), and four arms alternate in the same run at every k: nr_topk_dot at k (plain), nr_topk_dot at L (the
shortlist), nr_mmr_rerank alone on that shortlist, and a batched torch restatement of the re-ranking (gather, bmm Gram in fp32
with TF32 off, the k-step greedy, in chunks of --baseline-chunk users).  The MMR end to end is ops.top_k_scores(...,
mmr_lambda=, mmr_depth=): the shortlist plus the rerank.  Quality over a sample of users, plain lists against MMR lists: the
mean cosine of the pairs within a list, and the mean relevance (the score scaled to [0, 1] over the user's shortlist).  The
sampled MMR lists go through the fp64 path verifier of tests/mmr_ref.py.

DNN click scores (--scorer hifiark | dkn): nr_topk_archive, with and without a category cap (--max-per-category, default 2),
against a torch restatement and the per-user nr_archive_score_fwd path (tools/archive_pool_bench.py).

    python tools/recommend_bench.py [--users 700000] [--news 120000] [--dim 300] [--k 10 100] [--reps 3] [--seed 0]
                                    [--max-per-category M [--categories 17] [--zipf 0]]
                                    [--mmr-lambda X [--mmr-depth 40] [--stories 2000]]
                                    [--scorer {dot,hifiark,dkn} [--baseline-users 8192] [--sample-users 256]]

Time: CUDA events around the library's launches (operand planes, the top-k kernel, the split merge when there is one), after
a warm-up, best and median over reps.  Rates: multiply-adds of the three bf16 products per score (3 n_users n_news
round_up(D, 64)) over the time, and the bytes the design moves from HBM (fp32 inputs read once, hi/lo planes written once
and read once each: L2 serves the re-reads of the planes when the pool fits it, so this is a lower bound of DRAM traffic), plus
the outputs.  Prints the card name and power limit, then one JSON line.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "news-recommendation_b200", "src"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import archive_pool_bench  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except OSError:
        return "unknown card, power limit unknown"


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--users", type=int, default=700_000)
    ap.add_argument("--news", type=int, default=120_000)
    ap.add_argument("--dim", type=int, default=300)
    ap.add_argument("--k", type=int, nargs="+", default=[10, 100])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--baseline-chunk", type=int, default=8192, help="users per torch.matmul + torch.topk pass")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--max-per-category", type=int, default=None, metavar="M",
                    help="time nr_topk_dot_capped with this cap against nr_topk_dot")
    ap.add_argument("--categories", type=int, default=17, help="synthetic category keys (with --max-per-category)")
    ap.add_argument("--zipf", type=float, default=0.0, help="Zipf exponent of the category draw, 0: uniform")
    ap.add_argument("--mmr-lambda", type=float, default=None, metavar="X",
                    help="time nr_mmr_rerank at this lambda against nr_topk_dot and a torch restatement")
    ap.add_argument("--mmr-depth", type=int, default=40, metavar="L", help="shortlist length (with --mmr-lambda)")
    ap.add_argument("--stories", type=int, default=2000, help="story centroids of the clustered pool (with --mmr-lambda)")
    archive_pool_bench.add_args(ap)
    a = ap.parse_args(argv)
    if a.scorer != "dot":
        if a.mmr_lambda is not None:
            ap.error("--mmr-lambda is timed with --scorer dot")
        print(f"card: {card()}", flush=True)
        return archive_pool_bench.recommend_arms(a, card)
    if a.mmr_lambda is not None and (a.max_per_category is not None or not 0 <= a.mmr_lambda <= 1 or
                                     not max(a.k) <= a.mmr_depth <= 128):
        ap.error("--mmr-lambda takes a lambda in [0, 1], a --mmr-depth in [max(--k), 128] and no --max-per-category")
    if a.max_per_category is not None and (a.max_per_category < 1 or a.categories < 1):
        ap.error("--max-per-category and --categories must be at least 1")
    import torch
    from newsrec_b200 import require_cuda
    from newsrec_b200.ops import top_k_scores
    dev = require_cuda()
    torch.backends.cuda.matmul.allow_tf32 = False
    g = torch.Generator(device=dev).manual_seed(a.seed)
    users = torch.randn(a.users, a.dim, device=dev, generator=g)
    news = torch.randn(a.news, a.dim, device=dev, generator=g)
    print(f"card: {card()}", flush=True)
    if a.mmr_lambda is not None:
        news = news[torch.randint(0, a.stories, (a.news,), device=dev, generator=g) % a.news]
        news = news + 0.3 * torch.randn(a.news, a.dim, device=dev, generator=g)  # near-copies of a.stories stories
        return mmr(a, users, news, dev)
    if a.max_per_category is not None:
        return capped(a, users, news, dev)

    def kernel(k):
        return top_k_scores(users, news, k)

    def baseline(k):
        idx, sc = [], []
        for lo in range(0, a.users, a.baseline_chunk):
            s, i = torch.topk(users[lo:lo + a.baseline_chunk] @ news.T, k, dim=1)
            idx.append(i)
            sc.append(s)
        return torch.cat(idx), torch.cat(sc)

    def timed(fn, k):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        out = fn(k)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), out

    results = []
    Dp = (a.dim + 63) // 64 * 64
    for k in a.k:
        kernel(k), baseline(k)  # warm-up
        tk, tb = [], []
        for _ in range(a.reps):
            t, (ki, ks) = timed(kernel, k)
            tk.append(t)
            t, (bi, bs) = timed(baseline, k)
            tb.append(t)
        # cross-check on a sample of users against the fp32 baseline: scores within the bound, sets equal up to the bound
        rows = torch.linspace(0, a.users - 1, 2000, device=dev).long()
        u64, n64 = users[rows].double(), news.double()
        S = u64 @ n64.T
        E = (2.0 ** -15 + 3 * Dp * 2.0 ** -23) * (u64.abs() @ n64.abs().T)
        s_k, e_k = torch.gather(S, 1, ki[rows]), torch.gather(E, 1, ki[rows])
        score_ok = bool(((ks[rows].double() - s_k).abs() <= e_k).all())
        kth = torch.topk(S, k, dim=1).values[:, -1:]
        set_ok = bool((s_k >= kth - 2 * e_k).all())
        same = float((torch.sort(ki[rows], 1).values == torch.sort(bi[rows], 1).values).all(1).float().mean())
        mk, mb = sorted(tk)[len(tk) // 2], sorted(tb)[len(tb) // 2]
        fma = 3.0 * a.users * a.news * Dp
        ld = (a.dim + 7) // 8 * 8
        hbm = (a.users + a.news) * (4.0 * a.dim + 8.0 * ld) + 12.0 * a.users * k
        r = dict(k=k, kernel_ms_best=min(tk), kernel_ms_median=mk, baseline_ms_best=min(tb), baseline_ms_median=mb,
                 speedup_median=mb / mk, bf16_tflops=2 * fma / (mk * 1e-3) / 1e12, hbm_gb=hbm / 1e9,
                 hbm_tb_per_s=hbm / (mk * 1e-3) / 1e12, scores_within_bound=score_ok, set_within_bound=set_ok,
                 same_set_as_fp32_share=same)
        print(f"k={k}: nr_topk_dot {mk:.1f} ms (best {min(tk):.1f}), matmul+topk fp32 {mb:.1f} ms (best {min(tb):.1f}); "
              f"{r['bf16_tflops']:.0f} TFLOP/s of bf16 products; {r['hbm_gb']:.2f} GB of HBM traffic; checks "
              f"{score_ok and set_ok}; same set as fp32 for {same:.3f} of the sampled users", flush=True)
        results.append(r)
    print(json.dumps(dict(card=card(), users=a.users, news=a.news, dim=a.dim, reps=a.reps, results=results)))
    return 0


def capped(a, users, news, dev):
    """nr_topk_dot_capped against nr_topk_dot, alternating, at every k; prints one line per k and the JSON line."""
    import torch
    from newsrec_b200.ops import top_k_scores
    g = torch.Generator(device=dev).manual_seed(a.seed + 1)
    p = 1.0 / torch.arange(1, a.categories + 1, device=dev, dtype=torch.float64) ** a.zipf
    cat = torch.multinomial(p / p.sum(), a.news, replacement=True, generator=g).int()
    m = a.max_per_category
    Dp = (a.dim + 63) // 64 * 64

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), out

    results = []
    for k in a.k:
        run_c = lambda: top_k_scores(users, news, k, categories=cat, max_per_category=m)  # noqa: E731
        run_p = lambda: top_k_scores(users, news, k)  # noqa: E731
        run_c(), run_p()  # warm-up
        tc, tp = [], []
        for _ in range(a.reps):
            t, (ci, cs) = timed(run_c)
            tc.append(t)
            t, (pi, ps) = timed(run_p)
            tp.append(t)
        rows = torch.linspace(0, a.users - 1, 2000, device=dev).long()
        live = ci[rows] >= 0
        r = ci[rows].clamp(min=0)
        u64, n64 = users[rows].double(), news.double()
        s_k = (u64[:, None, :] * n64[r]).sum(-1)
        e_k = (2.0 ** -15 + 3 * Dp * 2.0 ** -23) * (u64.abs()[:, None, :] * n64[r].abs()).sum(-1)
        score_ok = bool(((cs[rows].double() - s_k).abs() <= e_k)[live].all())
        c = torch.where(live, cat[r].long(), -1 - torch.arange(k, device=dev))  # dead slots: distinct keys
        per_cat = (c[:, :, None] == c[:, None, :]).sum(-1)
        caps_ok = bool((per_cat[live] <= m).all())
        plain_ok = bool(torch.equal(ci, pi) and torch.equal(cs, ps)) if m >= k else None
        mc, mp = sorted(tc)[len(tc) // 2], sorted(tp)[len(tp) // 2]
        res = dict(k=k, capped_ms_best=min(tc), capped_ms_median=mc, plain_ms_best=min(tp), plain_ms_median=mp,
                   capped_over_plain=mc / mp, mean_returned=float((ci >= 0).sum(1).float().mean()),
                   scores_within_bound=score_ok, caps_obeyed=caps_ok, equal_to_plain=plain_ok)
        print(f"k={k} m={m} over {a.categories} categories (zipf {a.zipf}): nr_topk_dot_capped {mc:.1f} ms (best "
              f"{min(tc):.1f}), nr_topk_dot {mp:.1f} ms (best {min(tp):.1f}), {mc / mp:.2f}x; "
              f"{res['mean_returned']:.1f} news per user; checks {score_ok and caps_ok and plain_ok is not False}", flush=True)
        results.append(res)
    print(json.dumps(dict(card=card(), users=a.users, news=a.news, dim=a.dim, reps=a.reps, max_per_category=m,
                          categories=a.categories, zipf=a.zipf, results=results)))
    return 0


def torch_mmr(news, sl_idx, sl_score, k, lam, chunk):
    """The re-ranking restated in torch, chunk users at a time: (idx (U, k), score (U, k))."""
    import torch
    U, L = sl_idx.shape
    nn = torch.nn.functional.normalize(news, dim=1)
    out_i, out_s = [], []
    for lo in range(0, U, chunk):
        si, ss = sl_idx[lo:lo + chunk], sl_score[lo:lo + chunk]
        live = si >= 0
        X = nn[si.clamp(min=0)] * live[..., None]
        Gm = torch.bmm(X, X.transpose(1, 2))
        smax = torch.where(live, ss, -torch.inf).amax(1, keepdim=True)
        smin = torch.where(live, ss, torch.inf).amin(1, keepdim=True)
        rel = torch.where(smax == smin, torch.ones_like(ss), (ss - smin) / (smax - smin))
        msim = torch.zeros_like(ss)
        open_ = live.clone()
        rows = torch.arange(len(si), device=si.device)
        picks = []
        for t in range(k):
            obj = torch.where(open_, lam * rel - (1 - lam) * msim, -torch.inf)
            p = obj.argmax(1)  # the first maximum: the lower position
            ok = open_[rows, p]
            picks.append(torch.where(ok, p, -1))
            open_[rows, p] = False
            sim = Gm[rows, p]
            msim = sim if t == 0 else torch.maximum(msim, sim)
        P = torch.stack(picks, 1)
        out_i.append(torch.where(P >= 0, torch.gather(si, 1, P.clamp(min=0)), -1))
        out_s.append(torch.where(P >= 0, torch.gather(ss, 1, P.clamp(min=0)), -torch.inf))
    return torch.cat(out_i), torch.cat(out_s)


def mmr(a, users, news, dev):
    """nr_mmr_rerank against nr_topk_dot and the torch restatement, alternating, at every k; one line per k, the JSON line."""
    import torch
    from newsrec_b200 import load_library
    from newsrec_b200.ops import _p, _stream, top_k_scores
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import mmr_ref
    lib = load_library()
    L, lam = a.mmr_depth, a.mmr_lambda
    n, D = news.shape
    flag = torch.zeros(1, dtype=torch.int32, device=dev)

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), out

    results = []
    for k in a.k:
        sl = top_k_scores(users, news, L)
        idx = torch.empty((a.users, k), dtype=torch.int64, device=dev)
        score = torch.empty((a.users, k), dtype=torch.float32, device=dev)

        def rerank():
            rc = lib.nr_mmr_rerank(_p(news), n, D, D, _p(sl[0]), _p(sl[1]), a.users, L, k, lam, _p(idx), _p(score), _p(flag),
                                   _stream())
            assert rc == 0, lib.nr_last_error().decode()
            return idx, score
        arms = dict(plain=lambda: top_k_scores(users, news, k), shortlist=lambda: top_k_scores(users, news, L),
                    rerank=rerank, end_to_end=lambda: top_k_scores(users, news, k, mmr_lambda=lam, mmr_depth=L),
                    torch=lambda: torch_mmr(news, sl[0], sl[1], k, lam, a.baseline_chunk))
        times = {name: [] for name in arms}
        outs = {}
        for name, fn in arms.items():
            outs[name] = fn()  # warm-up
        for _ in range(a.reps):
            for name, fn in arms.items():
                t, outs[name] = timed(fn)
                times[name].append(t)
        med = {name: sorted(t)[len(t) // 2] for name, t in times.items()}
        same_e2e = bool(torch.equal(outs["end_to_end"][0], outs["rerank"][0]))
        agree_torch = float((outs["torch"][0] == outs["rerank"][0]).all(1).float().mean())
        # quality and the path verifier over a sample of users
        rows = torch.linspace(0, a.users - 1, 2000, device=dev).long()
        nn = torch.nn.functional.normalize(news.double(), dim=1)
        sl_i, sl_s = sl[0][rows], sl[1][rows].double()
        smax, smin = sl_s[:, :1], sl_s.min(1, keepdim=True).values

        def quality(i):
            X = nn[i.clamp(min=0)]
            C = torch.bmm(X, X.transpose(1, 2))
            off = ~torch.eye(k, dtype=torch.bool, device=dev)
            pos = (i[:, :, None] == sl_i[:, None, :]).float().argmax(2)
            rel = ((torch.gather(sl_s, 1, pos) - smin) / (smax - smin).clamp(min=1e-30))
            return float(C[:, off].mean()), float(rel.mean())
        cos_p, rel_p = quality(outs["plain"][0][rows])
        cos_m, rel_m = quality(outs["rerank"][0][rows])
        mmr_ref.verify_path(news.cpu().numpy(), sl_i.cpu().numpy(), sl[1][rows].cpu().numpy(), idx[rows].cpu().numpy(),
                            score[rows].cpu().numpy(), k, lam)
        gathered = a.users * L * D * 4.0
        res = dict(k=k, depth=L, mmr_lambda=lam, **{f"{name}_ms_median": m for name, m in med.items()},
                   **{f"{name}_ms_best": min(t) for name, t in times.items()},
                   rerank_row_gather_gb=gathered / 1e9, rerank_gather_tb_per_s=gathered / (med["rerank"] * 1e-3) / 1e12,
                   end_to_end_equals_rerank=same_e2e, torch_same_lists_share=agree_torch,
                   intra_list_cosine_plain=cos_p, intra_list_cosine_mmr=cos_m, relevance_plain=rel_p, relevance_mmr=rel_m,
                   path_verified=True)
        print(f"k={k} depth={L} lambda={lam}: nr_topk_dot@k {med['plain']:.1f} ms, nr_topk_dot@depth {med['shortlist']:.1f} "
              f"ms, nr_mmr_rerank {med['rerank']:.2f} ms, top_k_scores with MMR {med['end_to_end']:.1f} ms, torch "
              f"restatement {med['torch']:.1f} ms (same lists for {agree_torch:.3f} of users); intra-list cosine "
              f"{cos_p:.3f} plain / {cos_m:.3f} MMR, relevance {rel_p:.3f} / {rel_m:.3f}", flush=True)
        results.append(res)
    print(json.dumps(dict(card=card(), users=a.users, news=a.news, dim=a.dim, reps=a.reps, stories=a.stories,
                          results=results)))
    return 0


if __name__ == "__main__":
    sys.exit(main())
