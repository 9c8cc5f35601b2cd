"""Training-feed benchmark: the reference's loader (restated in oracle/feed_oracle.py, DataLoader with 4 workers and
pin_memory) against the device feed (newsrec_b200.feed), at batch 512 on synthetic parsed MIND of MIND-small size
(tools/make_synth_mind.py), for NRMS, NAML and LSTUR.

    python tools/feed_bench.py [--rows 150000] [--news 50000] [--runs 3] [--batches 30] [--steps 30] [--out result.json]

Per family it reports, each arm run --runs times with the two arms alternating:
  loader_ms     milliseconds per batch of the restated loader (host clock over --batches batches after a warm-up);
  feed_host_ms  host milliseconds of the device feed's next() (ends when the gather is enqueued);
  feed_gpu_ms   device milliseconds of the gather kernel itself (torch.profiler kernel records, a pass of its own), and
  feed_gpu_gbs  the bytes the gather has to move (gather_bytes, from the shapes) over that time;
  steps_per_s   a trainer-shaped loop (next(), forward, loss.item(), zero_grad, backward, Adam step) over --steps steps,
                once with each feed.
The card's name and power limit are read in the same run.  The data goes to a temporary directory.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "news-recommendation_b200", "src"), os.path.join(ROOT, "oracle")):
    sys.path.insert(0, p)

FAMILIES = ("NRMS", "NAML", "LSTUR")


def card():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[0] if q.returncode == 0 else None}


def config_for(fam, batch):
    import config as cfgmod
    return type(f"{fam}BenchConfig", (getattr(cfgmod, f"{fam}Config"),), {"batch_size": batch})


def reference_loader(ds, batch):
    from torch.utils.data import DataLoader
    return iter(DataLoader(ds, batch_size=batch, shuffle=True, num_workers=4, drop_last=True, pin_memory=True))


def time_loader(ds, batch, n):
    it = reference_loader(ds, batch)
    for _ in range(3):  # worker start-up and the first prefetches
        next(it)
    t0 = time.perf_counter()
    for _ in range(n):
        next(it)
    return (time.perf_counter() - t0) * 1e3 / n


def time_feed(feed, batch, n, epoch):
    """(host ms of next(), device ms of its gather kernel).  The host figure is a host clock around next() alone; the
    kernel's own time comes from a separate torch.profiler pass over n more batches (CUPTI kernel records), because
    CUDA events around next() would enclose the host work of next() as well: the stream is idle while it runs."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    it = iter(feed.loader(batch, shuffle=True, drop_last=True, epoch=epoch))
    next(it)
    torch.cuda.synchronize()
    host = 0.0
    for _ in range(n):
        t0 = time.perf_counter()
        next(it)
        host += time.perf_counter() - t0
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            next(it)
        torch.cuda.synchronize()
    # the mean over the kernel records the profiler kept (it can miss the first activity of a session)
    kernels = [e for e in prof.key_averages() if "feed_gather_kernel" in e.key]
    if len(kernels) != 1 or not n // 2 <= kernels[0].count <= n:
        raise RuntimeError(f"expected up to {n} feed_gather_kernel records, got {[(e.key, e.count) for e in kernels]}")
    return host * 1e3 / n, kernels[0].device_time_total / kernels[0].count / 1e3


def train_loop(fam, model, opt, it, steps):
    import torch
    y = None

    def step():
        nonlocal y
        mb = next(it)
        args = (mb["candidate_news"], mb["clicked_news"])
        out = model(mb["user"], mb["clicked_news_length"], *args) if fam == "LSTUR" else model(*args)
        if y is None:
            y = torch.zeros(out.shape[0], dtype=torch.long, device=out.device)
        loss = torch.nn.functional.cross_entropy(out, y)
        loss.item()
        opt.zero_grad()
        loss.backward()
        opt.step()

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        step()
    torch.cuda.synchronize()
    return steps / (time.perf_counter() - t0)


def bench_family(fam, data, args):
    import importlib
    import torch
    from feed_oracle import FeedOracle
    from newsrec_b200.feed import DeviceFeed
    cfg = config_for(fam, args.batch)
    beh, news = os.path.join(data, "behaviors_parsed.tsv"), os.path.join(data, "news_parsed.tsv")
    t0 = time.perf_counter()
    ref = FeedOracle(beh, news, cfg)
    t_ref = time.perf_counter() - t0
    t0 = time.perf_counter()
    feed = DeviceFeed(beh, news, cfg)
    torch.cuda.synchronize()
    t_feed = time.perf_counter() - t0
    # bytes one gather has to move: int32 table rows and behaviour entries in, int64 id blocks out, records in and out
    B, slots = args.batch, feed.H + feed.C
    ids = B * slots * sum(t.shape[1] for t in feed.news_tables.values())
    gather_bytes = ids * (4 + 8) + B * slots * 4 + B * 8 + B * (2 + feed.C) * (4 + 8)
    res = {"build_s": {"reference_loader": t_ref, "device_feed": t_feed}, "gather_bytes": gather_bytes,
           "loader_ms": [], "feed_host_ms": [], "feed_gpu_ms": [], "feed_gpu_gbs": [],
           "steps_per_s": {"reference_loader": [], "device_feed": []}}
    for r in range(args.runs):
        res["loader_ms"].append(time_loader(ref, args.batch, args.batches))
        h, g = time_feed(feed, args.batch, args.batches, r)
        res["feed_host_ms"].append(h)
        res["feed_gpu_ms"].append(g)
        res["feed_gpu_gbs"].append(gather_bytes / (g * 1e-3) / 1e9)
    torch.manual_seed(0)
    model = getattr(importlib.import_module("model." + fam), fam)(cfg).cuda().train()
    opt = torch.optim.Adam(model.parameters(), lr=cfg.learning_rate)
    for r in range(args.runs):
        res["steps_per_s"]["reference_loader"].append(train_loop(fam, model, opt, reference_loader(ref, args.batch), args.steps))
        res["steps_per_s"]["device_feed"].append(
            train_loop(fam, model, opt, iter(feed.loader(args.batch, shuffle=True, drop_last=True, epoch=100 + r)), args.steps))
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--rows", type=int, default=150000, help="behaviour rows (MIND-small's training split has ~157k impressions)")
    ap.add_argument("--news", type=int, default=50000, help="news (MIND-small: 51k)")
    ap.add_argument("--K", type=int, default=4)
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--batches", type=int, default=30)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--families", default=",".join(FAMILIES))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("feed_bench needs a CUDA device")
    out = {"card": card(), "args": vars(args), "families": {}}
    with tempfile.TemporaryDirectory() as tmp:
        subprocess.run([sys.executable, os.path.join(ROOT, "tools", "make_synth_mind.py"), tmp, str(args.rows), str(args.news), str(args.K)],
                       check=True, stdout=subprocess.DEVNULL)
        data = os.path.join(tmp, "data", "train")
        for fam in args.families.split(","):
            out["families"][fam] = bench_family(fam, data, args)
            print(fam, json.dumps(out["families"][fam]), flush=True)
    print(json.dumps(out))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
