"""Validation pass on the GPU: the device evaluator (newsrec_b200.evaluate) stage by stage against a restatement of the
reference evaluator's scoring loop (src/evaluate.py:243-271: one get_prediction + .tolist() per impression, then the
metrics of every impression on the host -- here the NumPy oracle in one process; the reference spreads sklearn calls over a
process pool).  Both paths score the same news / user vectors, in one process, on a validation set generated from a seed
and sized like MIND-small's (73 k impressions of ~37 candidates, 42 k news, 50 k users by default).

    python tools/eval_bench.py [--impressions 73152] [--candidates 37] [--news 42416] [--users 50000] [--seed 0]

Prints the card name and power limit next to the numbers, then one JSON line.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "news-recommendation_b200", "src"), os.path.join(ROOT, "oracle")):
    sys.path.insert(0, p)


def write_validation_set(d, n_imp, mean_cand, n_news, n_users, seed, T=20):
    rng = np.random.default_rng(seed)
    with open(os.path.join(d, "news_parsed.tsv"), "w") as f:
        f.write("id\tcategory\tsubcategory\ttitle\tabstract\ttitle_entities\tabstract_entities\n")
        titles = rng.integers(1, 70000, (n_news, T))
        lens = rng.integers(5, T + 1, n_news)
        for i in range(n_news):
            t = [int(x) for x in titles[i, :lens[i]]] + [0] * (T - lens[i])
            f.write(f"N{i}\t{rng.integers(1, 275)}\t{rng.integers(1, 275)}\t{t}\t{[0] * 50}\t{[0] * T}\t{[0] * 50}\n")
    hist = [" ".join(f"N{x}" for x in rng.integers(0, n_news, int(k))) for k in rng.integers(0, 80, n_users)]
    with open(os.path.join(d, "behaviors.tsv"), "w") as f:
        for i in range(n_imp):
            u = int(rng.integers(n_users))
            k = max(2, int(rng.poisson(mean_cand)))
            cand = rng.choice(n_news, k, replace=False)
            lab = (rng.random(k) < 0.04).astype(int)
            lab[int(rng.integers(k))] = 1
            f.write(f"{i + 1}\tU{u}\t11/15/2019 8:55:22 AM\t{hist[u]}\t{' '.join(f'N{c}-{y}' for c, y in zip(cand, lab))}\n")
    with open(os.path.join(d, "user2int.tsv"), "w") as f:
        f.write("user\tint\n" + "".join(f"U{i}\t{i + 1}\n" for i in range(n_users)))


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # the numbers are still printed; the card line says why it is missing
        return f"nvidia-smi unavailable ({e})"


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--impressions", type=int, default=73152)
    ap.add_argument("--candidates", type=int, default=37)
    ap.add_argument("--news", type=int, default=42416)
    ap.add_argument("--users", type=int, default=50000)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()

    import torch
    import config
    import ranking_metrics as R
    from model.NRMS import NRMS
    from newsrec_b200 import evaluate as E

    assert torch.cuda.is_available(), "eval_bench needs a CUDA device"
    torch.manual_seed(args.seed)
    model = NRMS(config.NRMSConfig).cuda().eval()
    sync = torch.cuda.synchronize

    def timed(fn):
        sync()
        t0 = time.perf_counter()
        out = fn()
        sync()
        return out, time.perf_counter() - t0

    with tempfile.TemporaryDirectory() as d, torch.no_grad():
        write_validation_set(d, args.impressions, args.candidates, args.news, args.users, args.seed)
        u2i = os.path.join(d, "user2int.tsv")
        E.evaluate(model, d, 4, 2000, user2int_path=u2i)  # warm-up: module loads, allocator, every kernel shape class
        t = {}
        (index, matrix), t["news"] = timed(lambda: E.news_matrix(model, d))
        tables, t["tables_host"] = timed(lambda: E.build_tables(d, index, config.NRMSConfig.num_clicked_news_a_user, user2int_path=u2i))
        flag = E.new_flag(matrix.device)
        users, t["users"] = timed(lambda: E.user_vectors(model, tables, matrix, flag))
        scores, t["scores"] = timed(lambda: E.impression_scores(tables, matrix, users, flag))
        means, t["metrics"] = timed(lambda: E.metric_means(scores, tables))
        _, t["evaluate_total"] = timed(lambda: E.evaluate(model, d, 4, user2int_path=u2i))

        # the reference's stage 3 + metrics on the same vectors
        offs, cand, seg_user = tables.seg_offsets, tables.cand, tables.seg_user

        def ref_scoring():
            preds = []
            for s in range(len(seg_user)):
                idx = cand[offs[s]:offs[s + 1]]
                cv = torch.stack([matrix[i] for i in idx], dim=0)
                preds.append(model.get_prediction(cv, users[seg_user[s]]).tolist())
            return preds

        preds, t["ref_scores"] = timed(ref_scoring)
        ref_means, t["ref_metrics"] = timed(lambda: np.nanmean(np.array(
            [R.single_impression(p, tables.labels[offs[s]:offs[s + 1]]) for s, p in enumerate(preds)]), axis=0))

    res = {"card": card(), "impressions": len(seg_user), "candidates": int(offs[-1]), "news": len(index) - 1,
           "distinct_histories": len(tables.user), "seconds": {k: round(v, 4) for k, v in t.items()},
           "device_scores_plus_metrics_s": round(t["scores"] + t["metrics"], 4),
           "reference_scores_plus_metrics_s": round(t["ref_scores"] + t["ref_metrics"], 4),
           "means_device": [float(x) for x in means], "means_reference_loop": [float(x) for x in ref_means],
           "max_abs_mean_diff": float(np.max(np.abs(np.array(means) - ref_means)))}
    print("card:", res["card"])
    for k, v in res["seconds"].items():
        print(f"  {k:16s} {v:9.4f} s")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
