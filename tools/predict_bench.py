"""Test-set predictions on the GPU, stage by stage: newsrec_b200.predict's chunked loop on a seeded synthetic test split
sized like MIND-large's (about 2.4 M impressions of ~37 candidates, as tools/eval_bench.py draws them), with NRMS at its
default config.  The host tables are drawn directly in NumPy (parsing behaviors.tsv is not timed); news_parsed.tsv is written
and encoded as predict() does.  Each stage ends in a device synchronise, so its time is the stage's own:

    news encoding (evaluate.news_matrix) | chunk tables (host) | user vectors | scoring | ranks | text | file write

The same run formats the ranks with a Python restatement (f"{id} [{','.join(map(str, r))}]\\n" per impression), times it,
and checks that both give the same bytes.

    python tools/predict_bench.py [--impressions 2400000] [--candidates 37] [--news 120000] [--users 1000000]
                                  [--chunk 32768] [--seed 0]

Prints the card name and power limit next to the numbers, then one JSON line.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "news-recommendation_b200", "src"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    sys.path.insert(0, p)


def write_news(d, n_news, rng, T=20):
    titles = rng.integers(1, 70000, (n_news, T))
    lens = rng.integers(5, T + 1, n_news)
    with open(os.path.join(d, "news_parsed.tsv"), "w") as f:
        f.write("id\tcategory\tsubcategory\ttitle\tabstract\ttitle_entities\tabstract_entities\n")
        for i in range(n_news):
            t = [int(x) for x in titles[i, :lens[i]]] + [0] * (T - lens[i])
            f.write(f"N{i}\t{rng.integers(1, 275)}\t{rng.integers(1, 275)}\t{t}\t{[0] * 50}\t{[0] * T}\t{[0] * 50}\n")


def draw_tables(n_imp, mean_cand, n_news, n_users, H, rng):
    """PredictTables of a synthetic test split: histories of 0..79 news (first H kept, left-padded), impressions of
    max(2, Poisson(mean_cand)) candidates (drawn with repeats, which change no work), impression ids 1..n_imp with random gaps."""
    from newsrec_b200.predict import PredictTables
    length = np.minimum(rng.integers(0, 80, n_users), H)
    history = np.full((n_users, H), n_news, np.int64)
    for k in range(1, H + 1):
        rows = length >= k
        history[rows, H - k] = rng.integers(0, n_news, int(rows.sum()))
    counts = np.maximum(2, rng.poisson(mean_cand, n_imp)).astype(np.int64)
    offsets = np.zeros(n_imp + 1, np.int64)
    offsets[1:] = np.cumsum(counts)
    cand = rng.integers(0, n_news, int(offsets[-1]))  # repeats within an impression do not change the work
    ids = np.cumsum(rng.integers(1, 3, n_imp)).astype(np.int64)
    return PredictTables(impression_id=ids, user=np.zeros(n_users, np.int64), history=history, history_length=length,
                         seg_user=rng.integers(0, n_users, n_imp), cand=cand, seg_offsets=offsets)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--impressions", type=int, default=2_400_000)
    ap.add_argument("--candidates", type=int, default=37)
    ap.add_argument("--news", type=int, default=120_000)
    ap.add_argument("--users", type=int, default=1_000_000)
    ap.add_argument("--chunk", type=int, default=32768)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()

    import torch
    import config
    from eval_bench import card
    from model.NRMS import NRMS
    from newsrec_b200 import evaluate as E
    from newsrec_b200.ops import impression_ranks, prediction_text

    assert torch.cuda.is_available(), "predict_bench needs a CUDA device"
    torch.manual_seed(args.seed)
    rng = np.random.default_rng(args.seed)
    model = NRMS(config.NRMSConfig).cuda().eval()
    H = config.NRMSConfig.num_clicked_news_a_user
    sync = torch.cuda.synchronize
    t = dict.fromkeys(["news_encoding", "chunk_tables_host", "user_vectors", "scoring", "ranks", "text", "file_write"], 0.0)

    def timed(key, fn):
        sync()
        t0 = time.perf_counter()
        out = fn()
        sync()
        t[key] += time.perf_counter() - t0
        return out

    with tempfile.TemporaryDirectory() as d, torch.no_grad():
        write_news(d, args.news, rng)
        tables = draw_tables(args.impressions, args.candidates, args.news, args.users, H, rng)
        # warm-up: module loads, allocator, every kernel shape class of a chunk
        _, matrix = E.news_matrix(model, d)
        warm = tables.chunk(0, min(args.chunk, args.impressions))
        flag, bad = E.new_flag(matrix.device), E.new_flag(matrix.device)
        seg = torch.from_numpy(warm.seg_offsets).cuda()
        prediction_text(torch.from_numpy(warm.impression_id), impression_ranks(
            E.impression_scores(warm, matrix, E.user_vectors(model, warm, matrix, flag), flag), seg, bad), seg)

        _, matrix = timed("news_encoding", lambda: E.news_matrix(model, d))
        S = args.impressions
        all_ranks = []
        out = os.path.join(d, "prediction.txt")
        with open(out, "wb") as f:
            for a in range(0, S, args.chunk):
                part = timed("chunk_tables_host", lambda: tables.chunk(a, min(S, a + args.chunk)))
                users = timed("user_vectors", lambda: E.user_vectors(model, part, matrix, flag))
                scores = timed("scoring", lambda: E.impression_scores(part, matrix, users, flag, model))
                seg = torch.from_numpy(part.seg_offsets).cuda()
                ranks = timed("ranks", lambda: impression_ranks(scores, seg, bad))
                text = timed("text", lambda: prediction_text(torch.from_numpy(part.impression_id), ranks, seg))
                timed("file_write", lambda: f.write(text.cpu().numpy().tobytes()))
                all_ranks.append(ranks.cpu().numpy())
        assert int(flag.item()) == 0 and int(bad.item()) == 0
        device_bytes = open(out, "rb").read()

        ranks = np.concatenate(all_ranks).tolist()
        ids, offs = tables.impression_id.tolist(), tables.seg_offsets.tolist()
        t0 = time.perf_counter()
        py_bytes = "".join(f"{i} [{','.join(map(str, ranks[offs[s]:offs[s + 1]]))}]\n" for s, i in enumerate(ids)).encode()
        t_py = time.perf_counter() - t0

    res = {"card": card(), "impressions": S, "candidates": int(tables.seg_offsets[-1]), "news": args.news,
           "histories": args.users, "chunk": args.chunk, "bytes": len(device_bytes), "bytes_equal": device_bytes == py_bytes,
           "seconds": {k: round(v, 4) for k, v in t.items()}, "device_stages_total_s": round(sum(t.values()), 4),
           "python_formatting_s": round(t_py, 4)}
    print("card:", res["card"])
    for k, v in res["seconds"].items():
        print(f"  {k:18s} {v:9.4f} s")
    print(f"  {'python_formatting':18s} {t_py:9.4f} s   (same bytes: {res['bytes_equal']})")
    print(json.dumps(res))
    if not res["bytes_equal"]:
        sys.exit(1)


if __name__ == "__main__":
    main()
