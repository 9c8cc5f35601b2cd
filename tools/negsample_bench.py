"""Negative-sampling benchmark: the device draw of the resampling feed (nr_sample_negatives, behind
newsrec_b200.feed.DeviceFeed(..., resample_negatives=True)) on seeded synthetic impressions shaped like MIND-large's
training split, against the reference's balancing loop.

    python tools/negsample_bench.py [--impressions 2200000] [--build-impressions 200000] [--K 2] [--draws 50] [--out result.json]

The impressions: lengths from a long-tailed log-normal (mean about 37 candidates, 2 to 300), 1 + Poisson(0.5) positives
(about 1.5, at most half the impression) in random places.  It reports:
  draw_ms          device milliseconds of one draw over --impressions impressions: CUDA events around --draws draws of new
                   epochs after --warmup draws;
  draw_bytes, draw_gbs  the bytes a draw has to move (labels read once, both offset arrays, the picked news rows read and
                   the candidate columns written) and that over draw_ms;
  checked_rows     rows of the first 20000 impressions compared with the NumPy oracle after the timed draws (must match);
  reference_s      host seconds of the restated reference balancing loop (oracle/negsample_oracle.py reference_balance,
                   one Python shuffle per impression) over the same impressions as token lists;
  build_s          host seconds of the feed's construction over a raw behaviors.tsv of --build-impressions impressions
                   (written to a temporary directory): parsing, the tables, the copy to the device and epoch 0's draw,
                   ending in a device synchronise.
The card's name and power limit are read in the same run.  Each stage rewrites --out, so a partial run keeps its numbers.
"""
import argparse
import json
import os
import random
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "news-recommendation_b200", "src"), os.path.join(ROOT, "oracle")):
    sys.path.insert(0, p)


def card():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[0] if q.returncode == 0 else None}


def write_data(out, n_imp, n_news, n_users, T=20, TA=50, seed=0):
    rng = np.random.default_rng(seed)
    with open(os.path.join(out, "news_parsed.tsv"), "w") as f:
        f.write("id\tcategory\tsubcategory\ttitle\tabstract\ttitle_entities\tabstract_entities\n")
        title, abstract = str([1] * T), str([1] * TA)
        f.writelines(f"N{i}\t1\t2\t{title}\t{abstract}\t{[0] * T}\t{[0] * TA}\n" for i in range(n_news))
    with open(os.path.join(out, "user2int.tsv"), "w") as f:
        f.write("user\tint\n")
        f.writelines(f"U{u}\t{u + 1}\n" for u in range(n_users))
    hist_len = rng.integers(0, 81, size=n_users)
    histories = [" ".join(f"N{x}" for x in rng.integers(0, n_news, size=n)) for n in hist_len]
    length = np.clip(np.rint(rng.lognormal(3.29, 0.8, size=n_imp)), 2, 300).astype(np.int64)
    pos = np.minimum(1 + rng.poisson(0.5, size=n_imp), length // 2)
    users = rng.integers(0, n_users, size=n_imp)
    news = rng.integers(0, n_news, size=int(length.sum()))
    off = np.concatenate([[0], np.cumsum(length)])
    # the first pos[i] candidates of a random order of each impression are its positives
    order = np.lexsort((rng.random(len(news)), np.repeat(np.arange(n_imp), length)))
    lab = np.zeros(len(news), np.int64)
    lab[order[(np.arange(len(news)) - np.repeat(off[:-1], length)) < np.repeat(pos, length)]] = 1
    token = np.asarray([[f"N{x}-0", f"N{x}-1"] for x in range(n_news)], dtype=object)[news, lab].tolist()
    with open(os.path.join(out, "behaviors.tsv"), "w") as f:
        for i in range(n_imp):
            f.write(f"{i + 1}\tU{users[i]}\t11/11/2019 9:00:00 AM\t{histories[users[i]]}\t{' '.join(token[off[i]:off[i + 1]])}\n")
    return {"impressions": n_imp, "candidates": int(length.sum()), "mean_candidates": float(length.mean()),
            "max_candidates": int(length.max()), "mean_positives": float(pos.mean())}


def synthetic_impressions(n_imp, n_news, seed=0):
    """(cand_rows int32, labels uint8, imp_offsets int64) shaped like MIND-large's training impressions (module docstring)."""
    rng = np.random.default_rng(seed)
    length = np.clip(np.rint(rng.lognormal(3.29, 0.8, size=n_imp)), 2, 300).astype(np.int64)
    pos = np.minimum(1 + rng.poisson(0.5, size=n_imp), length // 2)
    off = np.concatenate([[0], np.cumsum(length)])
    # the first pos[i] candidates of a random order of each impression are its positives
    order = np.argsort(np.repeat(np.arange(n_imp, dtype=np.float64), length) + rng.random(int(off[-1])))
    lab = np.zeros(int(off[-1]), np.uint8)
    lab[order[(np.arange(int(off[-1])) - np.repeat(off[:-1], length)) < np.repeat(pos, length)]] = 1
    return rng.integers(0, n_news, size=int(off[-1])).astype(np.int32), lab, off


def write_data(out, n_imp, n_news, n_users, T=20, TA=50, seed=0):
    """Raw behaviors.tsv (histories of 0 to 80 news per user), news_parsed.tsv and user2int.tsv for the feed's build."""
    rng = np.random.default_rng(seed + 1)
    with open(os.path.join(out, "news_parsed.tsv"), "w") as f:
        f.write("id\ttitle\n")
        f.writelines(f"N{i}\t{[1] * T}\n" for i in range(n_news))
    with open(os.path.join(out, "user2int.tsv"), "w") as f:
        f.write("user\tint\n")
        f.writelines(f"U{u}\t{u + 1}\n" for u in range(n_users))
    histories = [" ".join(f"N{x}" for x in rng.integers(0, n_news, size=n)) for n in rng.integers(0, 81, size=n_users)]
    users = rng.integers(0, n_users, size=n_imp)
    news, lab, off = synthetic_impressions(n_imp, n_news, seed)
    token = np.asarray([[f"N{x}-0", f"N{x}-1"] for x in range(n_news)], dtype=object)[news, lab].tolist()
    with open(os.path.join(out, "behaviors.tsv"), "w") as f:
        for i in range(n_imp):
            f.write(f"{i + 1}\tU{users[i]}\t11/11/2019 9:00:00 AM\t{histories[users[i]]}\t{' '.join(token[off[i]:off[i + 1]])}\n")


def log(res, out):
    print(json.dumps(res), flush=True)
    if out:
        os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
        with open(out, "w") as f:
            json.dump(res, f, indent=1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--impressions", type=int, default=2_200_000)
    ap.add_argument("--build-impressions", type=int, default=200_000)
    ap.add_argument("--news", type=int, default=100_000)
    ap.add_argument("--users", type=int, default=70_000)
    ap.add_argument("--K", type=int, default=2)
    ap.add_argument("--draws", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import ctypes as C
    import torch
    assert torch.cuda.is_available(), "negsample_bench needs a CUDA device"
    import config as cfgmod
    from negsample_oracle import balanced_rows, draw, reference_balance
    from newsrec_b200 import check, load_library
    from newsrec_b200.feed import DeviceFeed
    dev = torch.device("cuda", 0)
    res = {"card": card(), "K": a.K}

    cand, labels, off = synthetic_impressions(a.impressions, a.news)
    rows = balanced_rows(labels, off, a.K)
    row_offsets = np.concatenate([[0], np.cumsum(rows)]).astype(np.int64)
    R, H = int(row_offsets[-1]), 50
    res["data"] = {"impressions": a.impressions, "candidates": len(cand), "mean_candidates": len(cand) / a.impressions,
                   "max_candidates": int(np.diff(off).max()), "mean_positives": float(labels.sum()) / a.impressions, "rows": R}
    log(res, a.out)
    d = lambda x: torch.from_numpy(x).to(dev)
    dc, dl, do, dr = d(cand), d(labels), d(off), d(row_offsets)
    table = torch.zeros((R, H + 1 + a.K), dtype=torch.int32, device=dev)
    ptr = lambda t: C.c_void_p(t.data_ptr())
    lib, stream = load_library(), torch.cuda.current_stream(dev)
    run = lambda e: check(lib.nr_sample_negatives(ptr(dc), ptr(dl), ptr(do), a.impressions, ptr(dr), a.K, 1, e, ptr(table), H,
                                                  C.c_void_p(stream.cuda_stream)), "nr_sample_negatives")
    for e in range(a.warmup):
        run(e)
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for e in range(a.warmup, a.warmup + a.draws):
        run(e)
    end.record()
    end.synchronize()
    ms = start.elapsed_time(end) / a.draws
    nbytes = len(labels) + 2 * 8 * (a.impressions + 1) + 2 * 4 * R * (1 + a.K)
    res.update(draw_ms=ms, draw_bytes=nbytes, draw_gbs=nbytes / ms / 1e6)
    lim = min(a.impressions, 20000)
    ro, want = draw(cand[:off[lim]], labels[:off[lim]], off[:lim + 1], a.K, 1, a.warmup + a.draws - 1)
    assert np.array_equal(table[:ro[-1], H:].cpu().numpy(), want), "device draw differs from the oracle"
    res["checked_rows"] = int(ro[-1])
    log(res, a.out)

    rng, spent = random.Random(0), 0.0
    token = np.asarray([[f"N{x}-0", f"N{x}-1"] for x in range(a.news)], dtype=object)
    for lo in range(0, a.impressions, 100_000):
        hi = min(a.impressions, lo + 100_000)
        toks = token[cand[off[lo]:off[hi]], labels[off[lo]:off[hi]]].tolist()
        chunk = [toks[off[i] - off[lo]:off[i + 1] - off[lo]] for i in range(lo, hi)]
        t0 = time.perf_counter()
        reference_balance(chunk, a.K, rng)
        spent += time.perf_counter() - t0
    res["reference_s"] = spent
    log(res, a.out)

    cfg = type("NRMSBenchConfig", (cfgmod.NRMSConfig,), {"negative_sampling_ratio": a.K, "dataset_attributes": {"news": ["title"], "record": []}})
    with tempfile.TemporaryDirectory() as tmp:
        write_data(tmp, a.build_impressions, a.news, a.users)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        DeviceFeed(os.path.join(tmp, "behaviors_parsed.tsv"), os.path.join(tmp, "news_parsed.tsv"), cfg, device=dev,
                   resample_negatives=True, seed=1)
        torch.cuda.synchronize()
        res["build_impressions"], res["build_s"] = a.build_impressions, time.perf_counter() - t0
    log(res, a.out)


if __name__ == "__main__":
    main()
