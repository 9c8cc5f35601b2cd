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

NRMS, NAML, LSTUR, TANR and Exp1 score a user vector against a news vector by a dot product.  Hi-Fi Ark and DKN score them
with their DNN click predictor, over the user's archive (Hi-Fi Ark, similarity attention) or its one attention vector (DKN):
their models' ``pool_user_vector`` gives that operand and ``ops.top_k_scores(..., dnn=click_predictor.weights())``
(nr_topk_archive) the top k under the same scores ``evaluate`` computes, to within the bound of include/newsrec_b200.h.
A model of those two families without ``pool_user_vector`` is refused.

Diversified lists: with ``max_per_category=m`` no line holds more than m news of one category (``diversify_by="category"``)
or of one subcategory (``"subcategory"``), the column of ``news_parsed.tsv`` in the matrix's row order, copied once to the
device as int32.  The cap is applied inside the kernel (``ops.top_k_scores(..., categories=, max_per_category=)``,
nr_topk_dot_capped): the pool is walked best first and a news is taken iff fewer than m taken news share its category and
fewer than k are taken, so a line can be shorter than k when the caps run out.  One field per call.

Diversified by content: with ``mmr_lambda=lambda`` each line is the maximal-marginal-relevance re-ranking of the user's top
``mmr_depth`` news (default min(128, 4k)): k times, the shortlisted news not yet taken with the largest
lambda rel - (1 - lambda) max cosine to the news already taken, rel the click score scaled to [0, 1] over the shortlist and the
cosine that of the model's news vectors (``ops.top_k_scores(..., mmr_lambda=, mmr_depth=)``, nr_mmr_rerank).  lambda = 1 gives
the plain lines byte for byte; lower lambda trades relevance for lines that do not repeat one story.  Not together with a
category cap.

Live news only: with ``max_age_hours=H`` a line only holds news first shown in ``behaviors.tsv`` within H hours before the
line's request time, the time of the row ``evaluate.distinct_histories`` keeps for it (``window``: the definition, the
time order the device work runs in, and ties).  Each chunk's users are sorted by request time, so a block of 64 users
shares nearly one window and the kernels stream only its news tiles; the file does not depend on the chunk.  Caps, MMR and
every family work as above.

    python -m newsrec_b200.recommend --directory data/test --out recommendations.tsv [--k 10] [--keep-clicked]
                                     [--max-per-category M [--diversify-by {category,subcategory}]
                                      | --mmr-lambda X [--mmr-depth L]] [--max-age-hours H]
                                     [--checkpoint PATH | --checkpoint-dir DIR] [--user2int data/train/user2int.tsv]
                                     [--chunk-users N] [--set KNOB=VALUE ...]
"""
from __future__ import annotations

import os
import sys

import numpy as np

from . import NewsrecError, window
from .evaluate import _gather, distinct_histories, new_flag, news_matrix, read_behaviors, read_news, user_tables, user_vectors

DEFAULT_CHUNK = 65536
MAX_K = 128
DIVERSIFY_FIELDS = ("category", "subcategory")
# Families whose click score is not users . news: Hi-Fi Ark's depends on the candidate through the similarity attention over
# the user's archive; DKN's DNN scorer is separable (w2 . relu(W1c c + W1u u + b1)) but is not a single dot product.  They
# are served through the DNN scorer kernels when the model exposes pool_user_vector, and refused otherwise.
_REFUSED = {
    "HiFiArk": "Hi-Fi Ark's click score depends on the candidate through the similarity attention over the archive, so it is "
               "not a dot product of one user vector and one news vector",
    "DKN": "DKN's DNN click predictor is not a dot product of one user vector and one news vector",
}


def check_request(model, directory, k, max_per_category=None, diversify_by="category", mmr_lambda=None, mmr_depth=None,
                  who="recommend", max_age_hours=None):
    """Everything recommend() refuses, checked before any device work: k outside [1, 128], a cap that is not an integer >= 1,
    a diversify_by other than "category" / "subcategory", a family whose click predictor is not a dot product, an MMR
    request ops.mmr_request refuses or one together with a cap, a split without behaviors.tsv or news_parsed.tsv, (with
    a cap) a news_parsed.tsv without the diversify_by column, and (with max_age_hours) an age that is not a real number > 0
    or a behaviors.tsv time that does not parse.  Messages start with who.  Returns window.load's (W, behaviors, times), or
    None without max_age_hours."""
    if isinstance(k, bool) or not isinstance(k, (int, np.integer)) or not 1 <= k <= MAX_K:
        raise NewsrecError(f"{who}: k={k!r} must be an integer in [1, {MAX_K}]")
    if max_per_category is not None and (isinstance(max_per_category, bool) or
                                         not isinstance(max_per_category, (int, np.integer)) or max_per_category < 1):
        raise NewsrecError(f"{who}: max_per_category={max_per_category!r} must be an integer >= 1")
    if diversify_by not in DIVERSIFY_FIELDS:
        raise NewsrecError(f"{who}: diversify_by={diversify_by!r} must be one of {DIVERSIFY_FIELDS}")
    refuse_family(who, model)
    if max_age_hours is not None:
        window.max_age_seconds(who, max_age_hours)
    from .ops import mmr_request
    try:
        mmr = mmr_request(int(k), mmr_lambda, mmr_depth)
    except NewsrecError as e:
        raise NewsrecError(f"{who}: {e}") from None
    if mmr is not None and max_per_category is not None:
        raise NewsrecError(f"{who}: mmr_lambda and max_per_category do not combine")
    for f in ("behaviors.tsv", "news_parsed.tsv"):
        if not os.path.isfile(os.path.join(directory, f)):
            raise FileNotFoundError(f"{who}: {os.path.join(directory, f)} not found")
    if max_per_category is not None and diversify_by not in news_columns(directory):
        raise NewsrecError(f"{who}: {os.path.join(directory, 'news_parsed.tsv')} has no {diversify_by} column")
    return window.load(who, directory, max_age_hours)


def news_columns(directory):
    """The column names of directory/news_parsed.tsv."""
    with open(os.path.join(directory, "news_parsed.tsv")) as f:
        return f.readline().rstrip("\r\n").split("\t")


def list_options(who, directory, device, max_per_category=None, diversify_by="category", mmr_lambda=None, mmr_depth=None):
    """The keyword arguments of ops.top_k_scores that make recommend's lists: {} for the plain lists, the MMR knobs, or the
    category cap with the diversify_by column of news_parsed.tsv (in the matrix's row order) as int32 keys on device."""
    import torch
    if max_per_category is None:
        return {} if mmr_lambda is None else dict(mmr_lambda=mmr_lambda, mmr_depth=mmr_depth)
    keys = read_news(directory, [diversify_by])[1][diversify_by]
    if len(keys) and (keys.min() < -2 ** 31 or keys.max() >= 2 ** 31):
        raise NewsrecError(f"{who}: a {diversify_by} id does not fit in int32")
    return dict(categories=torch.from_numpy(keys.astype(np.int32)).to(device), max_per_category=int(max_per_category))


def time_ordered(pw, pool, opts):
    """The pool matrix and the top_k_scores keyword arguments of list_options in pw's time order (window): the matrix
    permuted by one gather, the category keys through pw.perm."""
    import torch
    perm = torch.from_numpy(pw.perm).to(pool.device)
    opts = dict(opts)
    if "categories" in opts:
        opts["categories"] = opts["categories"].index_select(0, perm)
    return pool.index_select(0, perm), opts


def refuse_family(who, model):
    """Raises NewsrecError for a model whose click score is not a dot product and that has no pool_user_vector."""
    name = type(model).__name__
    if name in _REFUSED and not hasattr(model, "pool_user_vector"):
        raise NewsrecError(f"{who}: {name} is not supported: {_REFUSED[name]}")


def pool_operands(model, tables, matrix, flag):
    """(users, dnn) for the whole-pool kernels: (user_vectors(...), None) for a dot-product family; for Hi-Fi Ark and DKN,
    model.pool_user_vector over batches of batch_size * 16 histories ((U, P, F) or (U, F)) and click_predictor.weights()."""
    import torch
    if type(model).__name__ not in _REFUSED:
        return user_vectors(model, tables, matrix, flag), None
    bs, H, F = model.config.batch_size * 16, tables.history.shape[1], matrix.shape[1]
    out = [model.pool_user_vector(_gather(tables.history[lo:lo + bs].reshape(-1), matrix, flag).view(-1, H, F))
           for lo in range(0, len(tables.user), bs)]
    users = torch.cat(out) if out else torch.zeros((0, F), dtype=torch.float32, device=matrix.device)
    return users, model.click_predictor.weights()


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
              chunk_users=DEFAULT_CHUNK, max_per_category=None, diversify_by="category", mmr_lambda=None, mmr_depth=None,
              max_age_hours=None) -> int:
    """Write the k best news of the pool for every distinct history of directory/behaviors.tsv to out_path; returns the
    number of lines.  Runs under torch.no_grad() on the model as given (call .eval() first).  The file appears only when
    every line is written; a non-finite score raises ValueError, a history row outside the news table IndexError.  With
    max_per_category=m a line holds at most m news of one diversify_by value; with mmr_lambda the lines are the MMR
    re-rankings of each user's top mmr_depth; with max_age_hours=H only news first shown within H hours before the line's
    request time are listed (module docstring)."""
    import torch
    from .ops import top_k_scores
    win = check_request(model, directory, k, max_per_category, diversify_by, mmr_lambda, mmr_depth,
                        max_age_hours=max_age_hours)
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
        cap = list_options("recommend", directory, matrix.device, max_per_category, diversify_by, mmr_lambda, mmr_depth)
        if win is not None:
            W, wbeh, times = win
            pw = window.pool_window(wbeh, times, news_ids)
            t_user = times[distinct_histories(wbeh).index.to_numpy()]
            pool, cap = time_ordered(pw, pool, cap)
        U = len(user)
        flag = new_flag(matrix.device)
        tmp = f"{out_path}.partial"
        try:
            with open(tmp, "wb") as f:
                for a in range(0, U, chunk_users):
                    b = min(U, a + chunk_users)
                    sel, row_range = slice(a, b), None
                    if win is not None:  # by request time within the chunk: a block of 64 users shares nearly one window
                        sel = a + np.argsort(t_user[a:b], kind="stable")
                        row_range = tuple(torch.from_numpy(x) for x in pw.ranges(t_user[sel], W))
                    users, dnn = pool_operands(model, _Users(user[sel], history[sel], length[sel]), matrix, flag)
                    excl = None, None
                    if exclude_clicked:
                        rows, offsets = exclusion_csr(history[sel], pad)
                        if win is not None:
                            rows = pw.to_time_order(rows)
                        excl = torch.from_numpy(rows), torch.from_numpy(offsets)
                    idx, _ = top_k_scores(users, pool, int(k), *excl, dnn=dnn, row_range=row_range, **cap)  # synchronises
                    if int(flag.item()):
                        raise IndexError("recommend: a history row is outside the news table")
                    idx = idx.cpu().numpy()
                    if win is not None:  # back to pool rows and to the users' order
                        idx[sel - a] = pw.to_rows(idx.copy())
                    f.write(format_lines(user_ids[a:b], idx, news_ids))
            os.replace(tmp, out_path)
        finally:
            if os.path.exists(tmp):
                os.remove(tmp)
    return U


def parse_args(argv=None):
    import argparse
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0],
                                 epilog="Every family is served: NRMS, NAML, LSTUR, TANR and Exp1 by the dot product of user and "
                                        "news vectors, Hi-Fi Ark and DKN by their DNN click predictor.")
    ap.add_argument("--directory", default="./data/test", help="split: news_parsed.tsv (the pool) and behaviors.tsv (the users)")
    ap.add_argument("--out", default="recommendations.tsv", help="the file to write")
    ap.add_argument("--k", type=int, default=10, help=f"news per user, 1 .. {MAX_K}")
    g = ap.add_mutually_exclusive_group()
    g.add_argument("--checkpoint", help="a checkpoint file (a dict with model_state_dict, as the trainer saves)")
    g.add_argument("--checkpoint-dir", help="load its latest ckpt-<n>.pth (default: ./checkpoint/<MODEL_NAME>)")
    ap.add_argument("--keep-clicked", action="store_true", help="let a user's clicked news be recommended back")
    add_diversify_args(ap, "category")
    add_window_arg(ap, "list only news first shown in behaviors.tsv within H hours before the line's request time "
                       "(inf: every news shown by then)")
    ap.add_argument("--user2int", default="./data/train/user2int.tsv")
    ap.add_argument("--chunk-users", type=int, default=DEFAULT_CHUNK, help="users scored per device pass")
    ap.add_argument("--set", action="append", default=[], metavar="KNOB=VALUE",
                    help="override a knob of the selected <MODEL_NAME>Config (repeatable)")
    args = ap.parse_args(argv)
    if not 1 <= args.k <= MAX_K:
        ap.error(f"--k must be in [1, {MAX_K}]")
    if args.chunk_users < 1:
        ap.error("--chunk-users must be at least 1")
    check_diversify_args(ap, args)
    check_window_arg(ap, args)
    return args


def add_window_arg(ap, help_text):
    """--max-age-hours H, shared with pool_eval; check_window_arg refuses what window.max_age_seconds refuses."""
    ap.add_argument("--max-age-hours", type=float, default=None, metavar="H", help=help_text)


def check_window_arg(ap, args):
    if args.max_age_hours is not None and not args.max_age_hours > 0.0:
        ap.error("--max-age-hours must be a number > 0 (inf: no age limit)")


def add_diversify_args(ap, diversify_by_default):
    """The list knobs of the command line, shared with pool_eval --lists: --max-per-category | --mmr-lambda, --diversify-by
    and --mmr-depth."""
    d = ap.add_mutually_exclusive_group()
    d.add_argument("--max-per-category", type=int, default=None, metavar="M",
                   help="at most M news of one category (see --diversify-by) per line")
    d.add_argument("--mmr-lambda", type=float, default=None, metavar="X",
                   help="re-rank each user's shortlist by maximal marginal relevance: X in [0, 1] weighs the click score "
                        "against similarity to the news already listed (1: the plain lines)")
    ap.add_argument("--diversify-by", choices=DIVERSIFY_FIELDS, default=diversify_by_default,
                    help="the news_parsed.tsv column --max-per-category caps")
    ap.add_argument("--mmr-depth", type=int, default=None, metavar="L",
                    help=f"shortlist length --mmr-lambda re-ranks, k .. {MAX_K} (default min({MAX_K}, 4k))")


def check_diversify_args(ap, args):
    """argparse errors for the knobs of add_diversify_args, given args.k."""
    if args.max_per_category is not None and args.max_per_category < 1:
        ap.error("--max-per-category must be at least 1")
    if args.mmr_lambda is not None and not 0.0 <= args.mmr_lambda <= 1.0:
        ap.error("--mmr-lambda must be in [0, 1]")
    if args.mmr_depth is not None:
        if args.mmr_lambda is None:
            ap.error("--mmr-depth needs --mmr-lambda")
        if not args.k <= args.mmr_depth <= MAX_K:
            ap.error(f"--mmr-depth must be in [--k, {MAX_K}]")


def main(argv=None):
    from .predict import load_model
    args = parse_args(argv)
    name, path, model = load_model(args.checkpoint, args.checkpoint_dir, args.set)
    n = recommend(model, args.directory, args.out, args.k, exclude_clicked=not args.keep_clicked, user2int_path=args.user2int,
                  chunk_users=args.chunk_users, max_per_category=args.max_per_category, diversify_by=args.diversify_by,
                  mmr_lambda=args.mmr_lambda, mmr_depth=args.mmr_depth, max_age_hours=args.max_age_hours)
    cap = "" if args.max_per_category is None else f" (at most {args.max_per_category} per {args.diversify_by})"
    if args.mmr_lambda is not None:
        cap = f" (MMR re-ranked, lambda {args.mmr_lambda})"
    if args.max_age_hours is not None:
        cap += f" (news at most {args.max_age_hours:g} h old)"
    print(f"{name} from {path}: top {args.k} news{cap} of {n} users written to {args.out}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
