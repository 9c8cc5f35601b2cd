"""Validation on the device: a drop-in for the reference's ``evaluate(model, directory, num_workers, max_count)``
(src/evaluate.py:171-271) with the same arguments and return value, ``(auc, mrr, ndcg5, ndcg10)`` as np.float64.

The reference keeps news and user vectors in Python dicts, scores one impression per ``get_prediction`` call followed by
a blocking ``.tolist()``, and computes the metrics with sklearn / NumPy once per impression in a process pool.  Here:

1. news      ``get_news_vector`` over the rows of news_parsed.tsv in the reference's batches, written into ONE fp32 device
             matrix (n_news + 1, D) whose last row is zeros (``PADDED_NEWS``);
2. users     one ``get_user_vector`` input per distinct history string (the reference's first-wins ``user2vector``),
             gathered on the device from that matrix;
3. scoring   every impression in one launch (``ops.predict_impressions``), then AUC / MRR / nDCG@5 / nDCG@10 of every
             impression in one launch (``ops.impression_metrics``), nanmean per column in fp64: one synchronisation.

The metrics follow the reference except where it is not well defined: among tied scores with different labels the
reference's MRR / nDCG depend on NumPy's unstable sort, here the stable reading of its expression is used (the later
candidate ranks first); an impression without negatives has AUC NaN and MRR / nDCG as computed (what scikit-learn 1.9
returns; older scikit-learn versions raised, which made the reference drop all four).  The host-side tables
(``build_tables``) need no CUDA.
"""
from __future__ import annotations

import sys
from ast import literal_eval
from dataclasses import dataclass
from os import path

import numpy as np

_LIST_COLUMNS = ("title", "abstract", "title_entities", "abstract_entities")


def read_news(directory, attributes, filename="news_parsed.tsv"):
    """news_parsed.tsv columns id + attributes (reference NewsDataset, evaluate.py:54-76): (ids list, {attr: int64 array})."""
    import pandas as pd
    df = pd.read_table(path.join(directory, filename), usecols=["id"] + list(attributes),
                       converters={a: literal_eval for a in set(attributes) & set(_LIST_COLUMNS)})
    cols = {a: np.asarray(df[a].tolist(), dtype=np.int64) for a in attributes}
    return df["id"].tolist(), cols


@dataclass
class EvalTables:
    """Everything stages 2 and 3 need, as row indices into the news matrix (pad row = n_news)."""
    user: np.ndarray            # (U,) int64 user2int of the first row holding each distinct history string (0 = unknown)
    history: np.ndarray         # (U, H) int64 news rows, left-padded with the pad row
    history_length: np.ndarray  # (U,) int64 number of real entries (<= H)
    seg_user: np.ndarray        # (S,) int64 the user row of every scored impression
    cand: np.ndarray            # (n_cand,) int64 candidate news rows, impressions back to back
    labels: np.ndarray          # (n_cand,) uint8
    seg_offsets: np.ndarray     # (S + 1,) int64


def _rows(news_index, ids):
    return [news_index[x] for x in ids]  # KeyError on an unknown news id, as the reference's news2vector[...]


def read_behaviors(directory, **kw):
    """behaviors.tsv as a DataFrame (columns impression_id, user, time, clicked_news, impressions); an empty history
    becomes ' ' (the reference's fillna).  kw goes to pandas.read_table."""
    import pandas as pd
    beh = pd.read_table(path.join(directory, "behaviors.tsv"), header=None, usecols=range(5),
                        names=["impression_id", "user", "time", "clicked_news", "impressions"], **kw)
    beh["clicked_news"] = beh["clicked_news"].fillna(" ")
    return beh


def distinct_histories(beh):
    """The (user, clicked_news) rows of beh (read_behaviors) that define the user tables: duplicate pairs dropped, then the
    first row of each distinct history string, in first-appearance order."""
    users = beh[["user", "clicked_news"]].drop_duplicates()
    return users[~users["clicked_news"].duplicated()]        # first-wins user2vector (evaluate.py:226-230)


def user_tables(beh, news_index, H, user2int_path):
    """The user half of build_tables: (user, history, history_length, hist_row) -- one row per distinct history string
    of beh (read_behaviors), hist_row mapping each string to its row."""
    import pandas as pd
    pad = news_index["PADDED_NEWS"]
    user2int = dict(pd.read_table(user2int_path).values.tolist())
    users = distinct_histories(beh)
    hist_row = {}
    U = len(users)
    user = np.zeros(U, np.int64)
    history = np.full((U, H), pad, np.int64)
    length = np.zeros(U, np.int64)
    for r, (u, hs) in enumerate(zip(users["user"].tolist(), users["clicked_news"].tolist())):
        hist_row[hs] = r
        user[r] = user2int.get(u, 0)
        ids = hs.split()[:H]
        length[r] = len(ids)
        if ids:
            history[r, H - len(ids):] = _rows(news_index, ids)
    return user, history, length, hist_row


def build_tables(directory, news_index, H, max_count=sys.maxsize, user2int_path="data/train/user2int.tsv"):
    """Host half of stages 2 and 3 (reference UserDataset / BehaviorsDataset and the loop at evaluate.py:243-265).

    news_index maps a news id to its matrix row and "PADDED_NEWS" to the zero row.  Users: behaviors.tsv columns 1 and 3,
    empty history -> ' ', duplicate (user, history) rows dropped; the FIRST row of each distinct history string defines its user (user2int, 0 if
    unknown) and its first H news ids.  Impressions: the first max_count - 1 rows (the reference increments its counter
    and breaks on count == max_count before scoring)."""
    beh = read_behaviors(directory)
    user, history, length, hist_row = user_tables(beh, news_index, H, user2int_path)
    n_imp = len(beh) if max_count < 1 else min(len(beh), max_count - 1)
    imp = beh.iloc[:n_imp]
    seg_user = np.asarray([hist_row[hs] for hs in imp["clicked_news"].tolist()], np.int64)
    cand, labels, offsets = impression_candidates(imp["impressions"], news_index)
    labels = np.where((labels >= 0) & (labels <= 1), labels, 2).astype(np.uint8)  # anything else is flagged on the device
    return EvalTables(user=user, history=history, history_length=length, seg_user=seg_user,
                      cand=cand, labels=labels, seg_offsets=offsets)


def impression_candidates(impressions, news_index):
    """The impressions column of read_behaviors ("N1-1 N2-0 ...") as CSR: (cand, labels, offsets) -- int64 news rows and
    labels as written, impressions back to back, and the (n_imp + 1,) int64 offsets."""
    cand, labels, counts = [], [], []
    for items in impressions.tolist():
        items = items.split()
        cand.extend(_rows(news_index, [x.split("-")[0] for x in items]))
        labels.extend(int(x.split("-")[1]) for x in items)
        counts.append(len(items))
    offsets = np.zeros(len(counts) + 1, np.int64)
    offsets[1:] = np.cumsum(counts)
    return np.asarray(cand, np.int64), np.asarray(labels, np.int64), offsets


def new_flag(device):
    """Device int32 flag the row gathers of stages 2 and 3 set on an out-of-range row (checked once, at the end)."""
    import torch
    return torch.zeros(1, dtype=torch.int32, device=device)


def _gather(ids, table, flag):
    """table[ids] through the library's fp32 row gather (nr_embedding_f32_fwd)."""
    import torch
    from .ops_cnn import EmbeddingF32Fn
    return EmbeddingF32Fn.apply(torch.from_numpy(np.ascontiguousarray(ids)).to(table.device), table, flag)


def news_matrix(model, directory):
    """Stage 1: (news_index, matrix) -- matrix (n_news + 1, D) fp32 on the device, the last row zeros (PADDED_NEWS);
    news_index maps each id to its row (the first row of an id wins, as in the reference's news2vector)."""
    import torch
    cfg = model.config
    attrs = cfg.dataset_attributes["news"]
    ids, cols = read_news(directory, attrs)
    n, bs = len(ids), cfg.batch_size * 16
    news_index = {}
    for i, x in enumerate(ids):
        news_index.setdefault(x, i)
    matrix = None
    for lo in range(0, n, bs):
        batch = {a: torch.from_numpy(cols[a][lo:lo + bs]) for a in attrs}  # what default_collate builds (int64)
        vec = model.get_news_vector(batch)
        if matrix is None:
            matrix = torch.zeros((n + 1, vec.shape[1]), dtype=torch.float32, device=vec.device)
        matrix[lo:lo + vec.shape[0]] = vec
    news_index["PADDED_NEWS"] = n
    return news_index, matrix


def user_vectors(model, tables, matrix, flag):
    """Stage 2: (U, D) user vectors, one per distinct history string, in batches of batch_size * 16."""
    import torch
    cfg = model.config
    bs, H = cfg.batch_size * 16, tables.history.shape[1]
    lstur = type(model).__name__ == "LSTUR"
    out = []
    for lo in range(0, len(tables.user), bs):
        hist = _gather(tables.history[lo:lo + bs].reshape(-1), matrix, flag).view(-1, H, matrix.shape[1])
        if lstur:
            out.append(model.get_user_vector(torch.from_numpy(tables.user[lo:lo + bs]),
                                             torch.from_numpy(tables.history_length[lo:lo + bs]), hist))
        else:
            out.append(model.get_user_vector(hist))
    if not out:
        return torch.zeros((0, matrix.shape[1]), dtype=torch.float32, device=matrix.device)
    return torch.cat(out)


def impression_scores(tables, matrix, users, flag, model=None):
    """Stage 3: (n_cand,) fp32 scores of every impression (at least one), one launch: nr_segment_dot for user vectors (U, D);
    for archives (U, P, D) (Hi-Fi Ark) the model's similarity-attention scorer against each impression's archive."""
    from .ops import predict_impressions
    cand, seg = _device_long(tables.cand, matrix), _device_long(tables.seg_offsets, matrix)
    if users.dim() == 3:
        per_imp = _gather(tables.seg_user, users.reshape(users.shape[0], -1), flag).view(-1, *users.shape[1:])
        return model.score_impressions(matrix, cand, seg, per_imp, flag)
    per_imp = _gather(tables.seg_user, users, flag)
    return predict_impressions(matrix, cand, seg, per_imp)


def _device_long(a, like):
    import torch
    return torch.from_numpy(a).to(like.device)


def metric_means(scores, tables):
    """(auc, mrr, ndcg5, ndcg10): nanmean over impressions, fp64, of the per-impression metrics (nr_impression_metrics)."""
    import torch
    from .ops import impression_metrics
    m = impression_metrics(scores, torch.from_numpy(tables.labels), _device_long(tables.seg_offsets, scores)).cpu().numpy()
    return tuple(np.float64(v) for v in np.nanmean(m, axis=0))


def evaluate(model, directory, num_workers, max_count=sys.maxsize, *, user2int_path="data/train/user2int.tsv"):
    """Reference src/evaluate.py:171-271 on the device.  num_workers is accepted for the signature and unused; runs under
    torch.no_grad() on the model as given (the trainer calls .eval() first)."""
    import torch
    with torch.no_grad():
        news_index, matrix = news_matrix(model, directory)
        tables = build_tables(directory, news_index, model.config.num_clicked_news_a_user, max_count, user2int_path)
        if len(tables.seg_user) == 0:  # max_count == 1 (the reference fails on its empty result)
            return (np.float64(np.nan),) * 4
        flag = new_flag(matrix.device)
        users = user_vectors(model, tables, matrix, flag)
        scores = impression_scores(tables, matrix, users, flag, model)
        means = metric_means(scores, tables)  # synchronises
        if int(flag.item()):
            raise IndexError("evaluate: a history or impression row is outside the news / user tables")
        return means
