"""nr_pool_ranks on the GPU at tools/recommend_bench.py's shape: the rank of every target of n_rows query rows among n_news news
(seeded synthetic fp32 vectors, D = 300 as NRMS's; 1 or 2 targets per row, 1.5 on average, and 0 to 50 exclusions), against
nr_topk_dot at k = 10 on the same rows and exclusions and against chunked torch.matmul in fp32 (TF32 off) plus a count of the
greater scores of every target, the three timed alternately in the same run.

    python tools/pool_rank_bench.py [--rows 700000] [--news 120000] [--dim 300] [--reps 3] [--seed 0]
                                    [--scorer {dot,hifiark,dkn} [--baseline-users 8192]]

--scorer hifiark | dkn times nr_pool_ranks_archive under the DNN click score instead, with nr_topk_archive at k = 10 and a
torch restatement (tools/archive_pool_bench.py).

Time: CUDA events around the library call alone (operand planes, the rank or top-k kernel, the split merge when there is one)
on device-resident CSR, after a warm-up, best and median over reps.  Check: on a sample of rows, the kernel's ranks and the
fp32 baseline's ranks both inside the band include/newsrec_b200.h states against fp64.  Prints the card name and power limit,
then one JSON line.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "news-recommendation_b200", "src"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import archive_pool_bench  # noqa: E402
from recommend_bench import card  # noqa: E402


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--rows", type=int, default=700_000)
    ap.add_argument("--news", type=int, default=120_000)
    ap.add_argument("--dim", type=int, default=300)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--baseline-chunk", type=int, default=4096, help="rows per torch.matmul + count pass")
    ap.add_argument("--sample", type=int, default=300, help="rows checked against the fp64 band")
    ap.add_argument("--seed", type=int, default=0)
    archive_pool_bench.add_args(ap)
    a = ap.parse_args(argv)
    if a.scorer != "dot":
        print(f"card: {card()}", flush=True)
        return archive_pool_bench.rank_arms(a, card)
    import torch
    from newsrec_b200 import check, load_library, require_cuda
    lib = load_library()
    dev = require_cuda()
    torch.backends.cuda.matmul.allow_tf32 = False
    g = torch.Generator(device=dev).manual_seed(a.seed)
    Q, n, D = a.rows, a.news, a.dim
    users = torch.randn(Q, D, device=dev, generator=g)
    news = torch.randn(n, D, device=dev, generator=g)
    n_t = 1 + (torch.rand(Q, device=dev, generator=g) < 0.5).long()
    t_off = torch.zeros(Q + 1, dtype=torch.int64, device=dev)
    t_off[1:] = torch.cumsum(n_t, 0)
    T = int(t_off[-1])
    t_row = torch.randint(0, n, (T,), device=dev, generator=g)
    second = torch.arange(T, device=dev) == t_off[:-1].repeat_interleave(n_t) + 1  # a row's two targets differ
    t_row[second] = (t_row[second.roll(-1)] + 1 + torch.randint(0, n - 1, (int(second.sum()),), device=dev, generator=g)) % n
    n_x = torch.randint(0, 51, (Q,), device=dev, generator=g)
    x_off = torch.zeros(Q + 1, dtype=torch.int64, device=dev)
    x_off[1:] = torch.cumsum(n_x, 0)
    x_row = torch.randint(0, n, (int(x_off[-1]),), device=dev, generator=g)
    print(f"card: {card()}", flush=True)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    ws_r = torch.empty(int(lib.nr_pool_ranks_workspace(Q, n, D)), dtype=torch.uint8, device=dev)
    ws_k = torch.empty(int(lib.nr_topk_dot_workspace(Q, n, D, 10)), dtype=torch.uint8, device=dev)
    rank = torch.empty(T, dtype=torch.int64, device=dev)
    score = torch.empty(T, dtype=torch.float32, device=dev)
    idx = torch.empty(Q, 10, dtype=torch.int64, device=dev)
    top = torch.empty(Q, 10, dtype=torch.float32, device=dev)
    flags = torch.zeros(3, dtype=torch.int32, device=dev)
    fl = [C.c_void_p(flags.data_ptr() + 4 * i) for i in range(3)]

    def ranks():
        check(lib.nr_pool_ranks(p(users), Q, D, p(news), n, D, D, p(t_off), p(t_row), p(x_off), p(x_row), p(rank), p(score),
                                *fl, p(ws_r), ws_r.numel(), stream), "nr_pool_ranks")

    def topk():
        check(lib.nr_topk_dot(p(users), Q, D, p(news), n, D, D, 10, p(x_off), p(x_row), p(idx), p(top), fl[0], fl[1], p(ws_k),
                              ws_k.numel(), stream), "nr_topk_dot")

    t_q = torch.arange(Q, device=dev).repeat_interleave(n_t)
    x_q = torch.arange(Q, device=dev).repeat_interleave(n_x)
    base_rank = torch.empty(T, dtype=torch.int64, device=dev)

    def baseline():
        for lo in range(0, Q, a.baseline_chunk):
            hi = min(Q, lo + a.baseline_chunk)
            S = users[lo:hi] @ news.T
            ta, tb = int(t_off[lo]), int(t_off[hi])
            xa, xb = int(x_off[lo]), int(x_off[hi])
            qt, rt = t_q[ta:tb] - lo, t_row[ta:tb]
            st = S[qt, rt]
            S[x_q[xa:xb] - lo, x_row[xa:xb]] = float("nan")  # exclusions and targets compare false
            S[qt, rt] = float("nan")
            Sq = S[qt]
            cols = torch.arange(n, device=dev)
            base_rank[ta:tb] = ((Sq > st[:, None]) | ((Sq == st[:, None]) & (cols[None, :] < rt[:, None]))).sum(1)

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    ranks(), topk(), baseline()  # warm-up
    tr, tk, tb = [], [], []
    for _ in range(a.reps):
        tr.append(timed(ranks))
        tk.append(timed(topk))
        tb.append(timed(baseline))
    assert flags.tolist() == [0, 0, 0], flags.tolist()
    # the band against fp64 on a sample of rows: kernel and fp32 baseline
    coeff = 2.0 ** -15 + 3 * ((D + 63) // 64 * 64) * 2.0 ** -23
    n64 = news.double()
    in_band_kernel = in_band_base = 0
    checked = 0
    for q in torch.linspace(0, Q - 1, a.sample).long().tolist():
        S = n64 @ users[q].double()
        E = coeff * (n64.abs() @ users[q].double().abs())
        elig = torch.ones(n, dtype=torch.bool, device=dev)
        elig[x_row[int(x_off[q]):int(x_off[q + 1])]] = False
        ts = t_row[int(t_off[q]):int(t_off[q + 1])]
        elig[ts] = False
        for j, t in enumerate(ts.tolist()):
            d, e = S - S[t], E + E[t]
            lo_, hi_ = int((elig & (d > e)).sum()), int((elig & (d >= -e)).sum())
            i = int(t_off[q]) + j
            in_band_kernel += lo_ <= int(rank[i]) <= hi_
            in_band_base += lo_ <= int(base_rank[i]) <= hi_
            checked += 1
    med = lambda x: sorted(x)[len(x) // 2]  # noqa: E731
    mr, mk, mb = med(tr), med(tk), med(tb)
    diff = (rank - base_rank).abs()
    r = dict(card=card(), rows=Q, news=n, dim=D, targets=T, exclusions=int(x_off[-1]), reps=a.reps,
             pool_ranks_ms_median=mr, pool_ranks_ms_best=min(tr), topk10_ms_median=mk, topk10_ms_best=min(tk),
             baseline_ms_median=mb, baseline_ms_best=min(tb), ratio_to_topk10=mr / mk, speedup_over_baseline=mb / mr,
             checked_targets=checked, kernel_in_band=in_band_kernel, baseline_in_band=in_band_base,
             ranks_equal_to_baseline_share=float((diff == 0).double().mean()), max_rank_difference=int(diff.max()))
    print(f"nr_pool_ranks {mr:.1f} ms (best {min(tr):.1f}), nr_topk_dot k=10 {mk:.1f} ms (best {min(tk):.1f}), "
          f"matmul+count fp32 {mb:.1f} ms (best {min(tb):.1f}); ratio to top-k {mr / mk:.2f}; band: kernel {in_band_kernel}/{checked}, "
          f"baseline {in_band_base}/{checked}; ranks equal to the baseline for {r['ranks_equal_to_baseline_share']:.4f}", flush=True)
    print(json.dumps(r))
    return 0


if __name__ == "__main__":
    sys.exit(main())
