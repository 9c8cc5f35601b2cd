"""Test-set predictions on the device: the leaderboard file of MIND's unlabeled test split, ``prediction.txt``, one line
``<impression_id> [r1,r2,...,rn]`` per impression, r_i the 1-based rank of candidate i among its impression's scores.

The reference cannot write it: its ``evaluate.py`` reads a label from every impression token (``N123-0``) and the test
split's tokens carry none (``N123``).  Here:

1. news      ``evaluate.news_matrix``, unchanged: one fp32 device matrix of every news vector;
2. tables    on the host, ``build_prediction_tables``: the user half of ``evaluate.build_tables`` (first-wins history
             strings) and the impressions with labelled or unlabelled tokens;
3. chunks    of ``chunk_impressions`` impressions: the user vectors of only the distinct histories the chunk references,
             its scores (``evaluate.impression_scores``), its ranks (``ops.impression_ranks``: the place the evaluator's
             metrics use, so MRR / nDCG recomputed from the file agree with ``evaluate``), its text
             (``ops.prediction_text``: line lengths, a scan and the bytes, on the device), appended to the file with one
             write.  Device memory is bounded by the chunk, not by the file, and the bytes do not depend on the chunk.

    python -m newsrec_b200.predict --directory data/test --out prediction.txt [--checkpoint PATH | --checkpoint-dir DIR]
                                   [--user2int data/train/user2int.tsv] [--set KNOB=VALUE ...]

loads ``<MODEL_NAME>`` from the drop-in's ``config`` / ``model`` packages and its latest ``ckpt-<n>.pth`` (as the
reference's ``evaluate.py`` does, one model: Exp1's ensemble is not loaded).
"""
from __future__ import annotations

import os
import re
import sys
from dataclasses import dataclass

import numpy as np

from .evaluate import impression_scores, new_flag, news_matrix, read_behaviors, user_tables, user_vectors

DEFAULT_CHUNK = 32768
_IMPRESSION_ID = re.compile(r"[0-9]+")


@dataclass
class PredictTables:
    """Stages 2 and 3 of a test split, as row indices into the news matrix (pad row = n_news); see evaluate.EvalTables."""
    impression_id: np.ndarray   # (S,) int64, non-negative
    user: np.ndarray            # (U,) int64
    history: np.ndarray         # (U, H) int64
    history_length: np.ndarray  # (U,) int64
    seg_user: np.ndarray        # (S,) int64
    cand: np.ndarray            # (n_cand,) int64
    seg_offsets: np.ndarray     # (S + 1,) int64

    def chunk(self, a, b):
        """Impressions [a, b) with only the users they reference (in row order)."""
        rows, inv = np.unique(self.seg_user[a:b], return_inverse=True)
        lo, hi = self.seg_offsets[a], self.seg_offsets[b]
        return PredictTables(impression_id=self.impression_id[a:b], user=self.user[rows], history=self.history[rows],
                             history_length=self.history_length[rows], seg_user=inv.reshape(-1).astype(np.int64),
                             cand=self.cand[lo:hi], seg_offsets=self.seg_offsets[a:b + 1] - lo)


def _impression_id(x, line):
    if not isinstance(x, str) or not _IMPRESSION_ID.fullmatch(x) or int(x) >= 1 << 63:
        raise ValueError(f"behaviors.tsv line {line}: impression id {x!r} is not a non-negative integer")
    return int(x)


def build_prediction_tables(directory, news_index, H, user2int_path="data/train/user2int.tsv"):
    """Host tables of a test split (behaviors.tsv of MIND's test set: tokens ``N123``; labelled tokens ``N123-1`` are
    accepted and their label ignored).  Users as evaluate.build_tables.  An unknown news id raises KeyError; an impression
    without candidates, or an impression id that is not a non-negative integer, raises ValueError naming the line."""
    beh = read_behaviors(directory, dtype={"impression_id": str, "impressions": str})
    user, history, length, hist_row = user_tables(beh, news_index, H, user2int_path)
    S = len(beh)
    ids = np.fromiter((_impression_id(x, r + 1) for r, x in enumerate(beh["impression_id"].tolist())), np.int64, S)
    seg_user = np.fromiter((hist_row[hs] for hs in beh["clicked_news"].tolist()), np.int64, S)
    tokens, counts = [], np.zeros(S, np.int64)
    for r, imp in enumerate(beh["impressions"].tolist()):
        items = imp.split() if isinstance(imp, str) else []
        if not items:
            raise ValueError(f"behaviors.tsv line {r + 1}: impression {ids[r]} has no candidate")
        counts[r] = len(items)
        tokens.extend(items)
    cand = np.fromiter((news_index[x.split("-", 1)[0]] for x in tokens), np.int64, len(tokens))  # KeyError: unknown news
    offsets = np.zeros(S + 1, np.int64)
    offsets[1:] = np.cumsum(counts)
    return PredictTables(impression_id=ids, user=user, history=history, history_length=length, seg_user=seg_user,
                         cand=cand, seg_offsets=offsets)


def predict(model, directory, out_path, *, user2int_path="data/train/user2int.tsv", chunk_impressions=DEFAULT_CHUNK) -> int:
    """Write prediction.txt of the impressions in directory/behaviors.tsv to out_path; returns the number of lines.  Runs
    under torch.no_grad() on the model as given (call .eval() first).  The file appears only when every line is written;
    a non-finite score raises ValueError, a history or candidate row outside the tables IndexError."""
    import torch
    from .ops import impression_ranks, prediction_text
    if chunk_impressions < 1:
        raise ValueError(f"predict: chunk_impressions={chunk_impressions}")
    with torch.no_grad():
        news_index, matrix = news_matrix(model, directory)
        tables = build_prediction_tables(directory, news_index, model.config.num_clicked_news_a_user, user2int_path)
        S = len(tables.impression_id)
        flag, bad = new_flag(matrix.device), new_flag(matrix.device)
        tmp = f"{out_path}.partial"
        try:
            with open(tmp, "wb") as f:
                for a in range(0, S, chunk_impressions):
                    part = tables.chunk(a, min(S, a + chunk_impressions))
                    users = user_vectors(model, part, matrix, flag)
                    scores = impression_scores(part, matrix, users, flag, model)
                    seg = torch.from_numpy(part.seg_offsets).to(matrix.device)
                    ranks = impression_ranks(scores, seg, bad)
                    text = prediction_text(torch.from_numpy(part.impression_id), ranks, seg)  # reads the total: synchronises
                    if int(flag.item()):
                        raise IndexError("predict: a history or impression row is outside the news / user tables")
                    if int(bad.item()):
                        s = int(torch.nonzero(ranks[seg[:-1]] == 0)[0])
                        raise ValueError(f"predict: impression {part.impression_id[s]} (behaviors.tsv line {a + s + 1}) has a "
                                         "non-finite score; its ranks are undefined")
                    f.write(text.cpu().numpy().tobytes())
            os.replace(tmp, out_path)
        finally:
            if os.path.exists(tmp):
                os.remove(tmp)
    return S


def latest_checkpoint(directory):
    """The ckpt-<n>.pth of directory with the largest n (the reference's train.latest_checkpoint), or None."""
    if not os.path.isdir(directory):
        return None
    found = {int(x.split(".")[-2].split("-")[-1]): x for x in os.listdir(directory)}
    return os.path.join(directory, found[max(found)]) if found else None


def load_checkpoint(path, device):
    """torch.load of a trainer checkpoint with weights only; its early_stop_value is a NumPy scalar, allowed explicitly."""
    import torch
    f64 = np.float64(0)
    with torch.serialization.safe_globals([f64.__reduce__()[0], np.dtype, type(f64.dtype)]):
        return torch.load(path, map_location=device, weights_only=True)


def load_model(checkpoint, checkpoint_dir, knobs):
    """(name, path, model): the drop-in's <MODEL_NAME> with the knobs applied, on the device in eval mode, loaded from
    checkpoint or the latest ckpt-<n>.pth of checkpoint_dir (default ./checkpoint/<MODEL_NAME>)."""
    import importlib
    src = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))  # the drop-in's config / model packages
    if src not in sys.path:
        sys.path.insert(0, src)
    from . import require_cuda
    from .launch import set_knobs
    cfgmod = importlib.import_module("config")
    name = cfgmod.model_name
    cfg = set_knobs(knobs)
    path = checkpoint or latest_checkpoint(checkpoint_dir or os.path.join("checkpoint", name))
    if path is None:
        raise SystemExit(f"no checkpoint file found in {checkpoint_dir or os.path.join('checkpoint', name)}")
    dev = require_cuda()
    model = getattr(importlib.import_module(f"model.{name}"), name)(cfg).to(dev)
    model.load_state_dict(load_checkpoint(path, dev)["model_state_dict"])
    model.eval()
    return name, path, model


def main(argv=None):
    import argparse
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--directory", default="./data/test", help="test split: news_parsed.tsv and behaviors.tsv")
    ap.add_argument("--out", default="prediction.txt", help="the file to write")
    g = ap.add_mutually_exclusive_group()
    g.add_argument("--checkpoint", help="a checkpoint file (a dict with model_state_dict, as the trainer saves)")
    g.add_argument("--checkpoint-dir", help="load its latest ckpt-<n>.pth (default: ./checkpoint/<MODEL_NAME>)")
    ap.add_argument("--user2int", default="./data/train/user2int.tsv")
    ap.add_argument("--chunk-impressions", type=int, default=DEFAULT_CHUNK, help="impressions scored per device pass")
    ap.add_argument("--set", action="append", default=[], metavar="KNOB=VALUE",
                    help="override a knob of the selected <MODEL_NAME>Config (repeatable)")
    args = ap.parse_args(argv)

    name, path, model = load_model(args.checkpoint, args.checkpoint_dir, args.set)
    n = predict(model, args.directory, args.out, user2int_path=args.user2int, chunk_impressions=args.chunk_impressions)
    print(f"{name} from {path}: {n} impressions written to {args.out}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
