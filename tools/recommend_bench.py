"""nr_topk_dot on the GPU at MIND-large's shape: the k best of n_news news for n_users users (seeded synthetic fp32 vectors,
D = 300 as NRMS's), against chunked torch.matmul in fp32 (TF32 off) + torch.topk over the same inputs, the two timed
alternately in the same run.  The baseline's answer also cross-checks the kernel's: every returned score within the bound of
include/newsrec_b200.h of the fp32 product, and the set equal up to news within twice the bound of the k-th best.

    python tools/recommend_bench.py [--users 700000] [--news 120000] [--dim 300] [--k 10 100] [--reps 3] [--seed 0]

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
    a = ap.parse_args(argv)
    import torch
    from newsrec_b200 import require_cuda
    from newsrec_b200.ops import top_k_scores
    dev = require_cuda()
    torch.backends.cuda.matmul.allow_tf32 = False
    g = torch.Generator(device=dev).manual_seed(a.seed)
    users = torch.randn(a.users, a.dim, device=dev, generator=g)
    news = torch.randn(a.news, a.dim, device=dev, generator=g)
    print(f"card: {card()}", flush=True)

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


if __name__ == "__main__":
    sys.exit(main())
