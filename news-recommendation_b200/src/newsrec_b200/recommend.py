"""Recommendations from the whole news pool on the device: for every user of a split, the k news of ``news_parsed.tsv``
with the highest click scores, one line ``<user_id>\\t<news_id>,<news_id>,...`` per user, best first.

``evaluate`` and ``predict`` only re-rank the candidates an impression log lists.  Here every user is scored against every
news without the U x n score matrix ever reaching memory (``ops.top_k_scores``, nr_topk_dot):

1. news      ``evaluate.news_matrix``: one fp32 device matrix of every news vector; the zero ``PADDED_NEWS`` row is not
             part of the pool;
2. users     one row per distinct history of ``behaviors.tsv`` (``evaluate.user_tables``, first-appearance order, the
             user of its first row), with ``exclude_clicked`` its history rows as the user's exclusion list;
3. chunks    of ``chunk_users`` users: their vectors (``evaluate.user_vectors``), their top k (``ops.top_k_scores``), the
             lines formatted on the host and appended to the file.  Device memory is bounded by the chunk and the pool,
             not by the file, and the bytes do not depend on the chunk.

The click predictor must be a dot product of a user vector and a news vector: NRMS, NAML, LSTUR, TANR and Exp1.

    python -m newsrec_b200.recommend --directory data/test --out recommendations.tsv [--k 10] [--keep-clicked]
                                     [--checkpoint PATH | --checkpoint-dir DIR] [--user2int data/train/user2int.tsv]
                                     [--chunk-users N] [--set KNOB=VALUE ...]
"""
from __future__ import annotations

import os
import sys

import numpy as np

from . import NewsrecError
from .evaluate import distinct_histories, new_flag, news_matrix, read_behaviors, read_news, user_tables, user_vectors

DEFAULT_CHUNK = 65536
MAX_K = 128
# Families whose click score is not users . news: Hi-Fi Ark's depends on the candidate through the similarity attention over
# the user's archive; DKN's DNN scorer is separable (w2 . relu(W1c c + W1u u + b1)) but is not a single dot product.
_REFUSED = {
    "HiFiArk": "Hi-Fi Ark's click score depends on the candidate through the similarity attention over the archive, so it is "
               "not a dot product of one user vector and one news vector",
    "DKN": "DKN's DNN click predictor is not a dot product of one user vector and one news vector",
}


def check_request(model, directory, k):
    """Everything recommend() refuses, checked before any device work: k outside [1, 128], a family whose click predictor is
    not a dot product, a split without behaviors.tsv or news_parsed.tsv."""
    if isinstance(k, bool) or not isinstance(k, (int, np.integer)) or not 1 <= k <= MAX_K:
        raise NewsrecError(f"recommend: k={k!r} must be an integer in [1, {MAX_K}]")
    name = type(model).__name__
    if name in _REFUSED:
        raise NewsrecError(f"recommend: {name} is not supported: {_REFUSED[name]}")
    for f in ("behaviors.tsv", "news_parsed.tsv"):
        if not os.path.isfile(os.path.join(directory, f)):
            raise FileNotFoundError(f"recommend: {os.path.join(directory, f)} not found")


def exclusion_csr(history, pad):
    """(rows, offsets) of history (U, H) int64 news rows: each user's rows other than the padding row pad, in order, as CSR
    (offsets (U + 1,) int64).  A news clicked twice appears twice, which the kernel treats as one exclusion."""
    history = np.asarray(history, np.int64)
    keep = history != pad
    offsets = np.zeros(len(history) + 1, np.int64)
    offsets[1:] = np.cumsum(keep.sum(axis=1))
    return history[keep], offsets


def format_lines(user_ids, idx, news_ids):
    """The bytes of one line per user: "<user_id>\\t<news_id>,<news_id>,...\\n", the ids of idx's rows in order, -1 slots left
    out."""
    out = []
    for u, row in zip(user_ids, idx.tolist()):
        out.append(f"{u}\t" + ",".join(news_ids[r] for r in row if r >= 0) + "\n")
    return "".join(out).encode()


class _Users:
    """The user tables of a chunk, as evaluate.user_vectors reads them."""

    def __init__(self, user, history, history_length):
        self.user, self.history, self.history_length = user, history, history_length


def recommend(model, directory, out_path, k=10, *, exclude_clicked=True, user2int_path="data/train/user2int.tsv",
              chunk_users=DEFAULT_CHUNK) -> int:
    """Write the k best news of the pool for every distinct history of directory/behaviors.tsv to out_path; returns the
    number of lines.  Runs under torch.no_grad() on the model as given (call .eval() first).  The file appears only when
    every line is written; a non-finite score raises ValueError, a history row outside the news table IndexError."""
    import torch
    from .ops import top_k_scores
    check_request(model, directory, k)
    if chunk_users < 1:
        raise ValueError(f"recommend: chunk_users={chunk_users}")
    with torch.no_grad():
        news_index, matrix = news_matrix(model, directory)
        pad = news_index["PADDED_NEWS"]
        news_ids = read_news(directory, [])[0]
        beh = read_behaviors(directory)
        user_ids = distinct_histories(beh)["user"].tolist()
        user, history, length, _ = user_tables(beh, news_index, model.config.num_clicked_news_a_user, user2int_path)
        pool = matrix[:pad]
        U = len(user)
        flag = new_flag(matrix.device)
        tmp = f"{out_path}.partial"
        try:
            with open(tmp, "wb") as f:
                for a in range(0, U, chunk_users):
                    b = min(U, a + chunk_users)
                    users = user_vectors(model, _Users(user[a:b], history[a:b], length[a:b]), matrix, flag)
                    excl = None, None
                    if exclude_clicked:
                        rows, offsets = exclusion_csr(history[a:b], pad)
                        excl = torch.from_numpy(rows), torch.from_numpy(offsets)
                    idx, _ = top_k_scores(users, pool, int(k), *excl)  # reads its flags: synchronises
                    if int(flag.item()):
                        raise IndexError("recommend: a history row is outside the news table")
                    f.write(format_lines(user_ids[a:b], idx.cpu().numpy(), news_ids))
            os.replace(tmp, out_path)
        finally:
            if os.path.exists(tmp):
                os.remove(tmp)
    return U


def parse_args(argv=None):
    import argparse
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--directory", default="./data/test", help="split: news_parsed.tsv (the pool) and behaviors.tsv (the users)")
    ap.add_argument("--out", default="recommendations.tsv", help="the file to write")
    ap.add_argument("--k", type=int, default=10, help=f"news per user, 1 .. {MAX_K}")
    g = ap.add_mutually_exclusive_group()
    g.add_argument("--checkpoint", help="a checkpoint file (a dict with model_state_dict, as the trainer saves)")
    g.add_argument("--checkpoint-dir", help="load its latest ckpt-<n>.pth (default: ./checkpoint/<MODEL_NAME>)")
    ap.add_argument("--keep-clicked", action="store_true", help="let a user's clicked news be recommended back")
    ap.add_argument("--user2int", default="./data/train/user2int.tsv")
    ap.add_argument("--chunk-users", type=int, default=DEFAULT_CHUNK, help="users scored per device pass")
    ap.add_argument("--set", action="append", default=[], metavar="KNOB=VALUE",
                    help="override a knob of the selected <MODEL_NAME>Config (repeatable)")
    args = ap.parse_args(argv)
    if not 1 <= args.k <= MAX_K:
        ap.error(f"--k must be in [1, {MAX_K}]")
    if args.chunk_users < 1:
        ap.error("--chunk-users must be at least 1")
    return args


def main(argv=None):
    from .predict import load_model
    args = parse_args(argv)
    name, path, model = load_model(args.checkpoint, args.checkpoint_dir, args.set)
    n = recommend(model, args.directory, args.out, args.k, exclude_clicked=not args.keep_clicked, user2int_path=args.user2int,
                  chunk_users=args.chunk_users)
    print(f"{name} from {path}: top {args.k} news of {n} users written to {args.out}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
