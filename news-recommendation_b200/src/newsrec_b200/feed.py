"""Device-resident training feed (SURVEY.md section 8f, row N3): a drop-in for the reference's ``BaseDataset`` plus its
``DataLoader`` whose batches are gathered on the device.

``DeviceFeed(behaviors_path, news_path)`` parses news_parsed.tsv and behaviors_parsed.tsv once into int32 tables:

* one news table per attribute of ``config.dataset_attributes["news"]``, (n_news + 1, L) with L = num_words_title /
  num_words_abstract for the list fields and 1 for category / subcategory; the last row is the all-zero padding news;
* the behaviour table (R, H + C): the news rows of the first H = num_clicked_news_a_user browsed news of every row,
  left-padded with the padding row, then its C = 1 + K candidates;
* the per-row records (R, 2 + C): user, clicked_news_length (the history length after truncation), the C clicked labels.

``DeviceFeed.loader(batch_size, shuffle, drop_last)`` iterates batches in the reference's minibatch format.  Each ``next()``
slices the epoch's row permutation (held on the device) and makes ONE launch (``nr_feed_gather``) on the feed device's current stream that
writes every field's impression-major id block -- the layout ``SlotPacker.pack`` produces from a collated batch -- and the
records.  ``clicked_news`` / ``candidate_news`` are ``FeedSlots``: slot-major lists of dicts of (B, L) views into those
blocks, so code that reads a slot tensor sees the reference loader's values (on the device), and ``SlotPacker.pack`` hands
the blocks to the encoders without another launch.

Row order: a ``DistributedSampler`` over the rows with a seed and an epoch counter (``newsrec_b200.launch --device-feed``
advances the epoch each time the trainer re-creates its loader), with one replica at world size 1.  This is another random
stream than the reference's ``RandomSampler``, with the same distribution.

Negatives redrawn every epoch: ``DeviceFeed(behaviors_path, news_path, config, resample_negatives=True, seed=s)`` reads
MIND's raw behaviors.tsv from behaviors_path's directory (users through user2int.tsv) instead of behaviors_parsed.tsv.  Its
rows are the reference's balancing (parse_behaviors): impression i owns min(P, N // K) rows, row p holding the p-th positive
and K negatives no other row of the impression holds.  The history columns and the records [user, clicked_news_length,
1, 0, ..., 0] are written once; ``loader(..., epoch=e)`` redraws the candidate columns for (s, e) with ONE launch
(``nr_sample_negatives``) on the stream the gathers use, before its first batch.  The table holds epoch 0's draw from
construction on; ``behaviors`` and ``feed[idx]`` read the current draw back from the device.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass

import numpy as np
import torch
from torch.utils.data import Dataset

_LIST_FIELDS = ("title", "abstract", "title_entities", "abstract_entities")
_NEWS_FIELDS = ("category", "subcategory") + _LIST_FIELDS
_RECORDS = ("user", "clicked_news_length")  # then the C clicked labels


def _field_width(config, attr):
    if attr in ("title", "title_entities"):
        return int(config.num_words_title)
    if attr in ("abstract", "abstract_entities"):
        return int(config.num_words_abstract)
    return 1


def _int32(a, what):
    a = np.asarray(a, dtype=np.int64)
    if a.size and (a.min() < np.iinfo(np.int32).min or a.max() > np.iinfo(np.int32).max):
        raise ValueError(f"{what}: values outside int32")
    return np.ascontiguousarray(a, dtype=np.int32)


def _default_config():
    import importlib
    cfgmod = importlib.import_module("config")
    return getattr(cfgmod, f"{cfgmod.model_name}Config")


class FeedSlots(list):
    """Slot-major list of per-slot dicts of (B, L) views (category / subcategory: (B,)) into `blocks`, the batch's
    impression-major int64 id blocks {field: (B*H + B*C, L)}; `clicked_news` and `candidate_news` of one batch share them."""

    def __init__(self, slots, blocks, B):
        super().__init__(slots)
        self.blocks, self.B = blocks, B


class DeviceFeed(Dataset):
    """The reference BaseDataset's constructor signature and length; the tables are parsed once (host arrays
    `news_tables`, `behaviors`, `records`) and copied to `device` (default: the current CUDA device, if any).
    resample_negatives: rows from the raw behaviors.tsv beside behaviors_path, negatives drawn on the device per (seed,
    epoch) (module docstring); user2int_path defaults to the user2int.tsv beside it.  Such a feed needs a CUDA device."""

    def __init__(self, behaviors_path, news_path, config=None, device=None, *, resample_negatives=False, user2int_path=None, seed=0):
        import pandas as pd
        from .evaluate import read_news
        super().__init__()
        self.config = config = config if config is not None else _default_config()
        self.attributes = list(config.dataset_attributes["news"])
        self.record_names = list(config.dataset_attributes["record"])
        for a in self.attributes:
            if a not in _NEWS_FIELDS:
                raise ValueError(f"unknown news attribute {a!r}")
        for r in self.record_names:
            if r not in _RECORDS:
                raise ValueError(f"unknown record {r!r}")
        H = self.H = int(config.num_clicked_news_a_user)

        try:
            ids, cols = read_news(os.path.dirname(news_path), self.attributes, os.path.basename(news_path))
        except ValueError as e:  # np.asarray over list cells of different lengths
            raise ValueError(f"{news_path}: a list column has rows of different lengths ({e})") from e
        index = {}
        for i, x in enumerate(ids):
            if x in index:
                raise ValueError(f"{news_path}: news id {x!r} appears more than once")
            index[x] = i
        pad = self.pad_row = len(ids)
        self.news_tables = {}
        for a in self.attributes:
            L = _field_width(config, a)
            col = cols[a].reshape(len(ids), -1)
            if col.shape[1] != L:
                raise ValueError(f"{news_path}: column {a!r} has {col.shape[1]} entries per news, the config says {L}")
            self.news_tables[a] = _int32(np.concatenate([col, np.zeros((1, L), np.int64)]), a)

        self.resample_negatives, self.seed, self.epoch = bool(resample_negatives), int(seed), 0
        self._stale = False  # the device table holds a draw the host copy does not
        if self.resample_negatives:
            directory = os.path.dirname(behaviors_path)
            self.K = int(config.negative_sampling_ratio)
            self.impressions = resample_tables(directory, dict(index, PADDED_NEWS=pad), H, self.K,
                                               user2int_path or os.path.join(directory, "user2int.tsv"))
            self.C = 1 + self.K
            self._behaviors, self.records = self.impressions.behaviors, self.impressions.records
        else:
            self._parse_balanced(pd.read_table(behaviors_path), behaviors_path, index, pad)

        if device is None and torch.cuda.is_available():
            device = torch.device("cuda", torch.cuda.current_device())
        self.device = torch.device(device) if device is not None else None
        if self.device is not None and self.device.type == "cuda" and self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self._dev = None
        if self.device is not None and self.device.type == "cuda":
            to = lambda a: torch.from_numpy(a).to(self.device)
            self._dev = {"news": {a: to(t) for a, t in self.news_tables.items()}, "behaviors": to(self._behaviors),
                         "records": to(self.records)}
        if self.resample_negatives:
            if self._dev is None:
                from . import NewsrecError
                raise NewsrecError("DeviceFeed(resample_negatives=True) needs a CUDA device: the negatives are drawn there only")
            t = self.impressions
            self._dev.update(cand_rows=to(t.cand_rows), labels=to(t.labels), imp_offsets=to(t.imp_offsets), row_offsets=to(t.row_offsets))
            self.epoch = None
            self.draw(0)

    def _parse_balanced(self, beh, behaviors_path, index, pad):
        """behaviors_parsed.tsv rows (user, clicked_news, candidate_news, clicked) -> self.behaviors, self.records, self.C."""
        H, R, C = self.H, len(beh), None
        behaviors, records = [], []
        for r, (user, hist, cand, clicked) in enumerate(zip(beh["user"].tolist(), beh["clicked_news"].tolist(),
                                                            beh["candidate_news"].tolist(), beh["clicked"].tolist())):
            h = hist.split()[:H]
            c = cand.split()
            labels = [int(x) for x in clicked.split()]
            if C is None:
                C = len(c)
            if len(c) != C or len(labels) != C:
                raise ValueError(f"{behaviors_path}: row {r} has {len(c)} candidates and {len(labels)} labels, row 0 has {C}: "
                                 "a batch needs the same number in every row")
            behaviors.append([pad] * (H - len(h)) + [index[x] for x in h] + [index[x] for x in c])  # KeyError: unknown news id
            records.append([int(user), len(h)] + labels)
        if C is None or C < 1:
            raise ValueError(f"{behaviors_path}: no behaviour rows with candidates")
        self.C = C
        self._behaviors = _int32(np.asarray(behaviors, np.int64).reshape(R, H + C), "behaviour table")
        self.records = _int32(np.asarray(records, np.int64).reshape(R, 2 + C), "user / clicked columns")

    @property
    def behaviors(self):
        """The behaviour table (R, H + C) int32 on the host; a resampling feed's candidate columns hold the current draw."""
        if self._stale:
            self._behaviors = self._dev["behaviors"].cpu().numpy()
            self._stale = False
        return self._behaviors

    def draw(self, epoch):
        """Redraw a resampling feed's candidate columns for (self.seed, epoch): one nr_sample_negatives launch on the feed
        device's current stream, none when the table already holds that epoch."""
        if epoch == self.epoch:
            return
        from . import check, load_library
        d, t = self._dev, self.impressions
        ptr = lambda x: C.c_void_p(x.data_ptr())
        with torch.cuda.device(self.device):
            check(load_library().nr_sample_negatives(ptr(d["cand_rows"]), ptr(d["labels"]), ptr(d["imp_offsets"]), len(t.imp_offsets) - 1,
                                                     ptr(d["row_offsets"]), self.K, self.seed & 0xFFFFFFFFFFFFFFFF, int(epoch),
                                                     ptr(d["behaviors"]), self.H, C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)),
                  "nr_sample_negatives")
        self.epoch, self._stale = epoch, True

    def __len__(self):
        return len(self._behaviors)

    def __getitem__(self, idx):
        """Row idx in the reference dataset's item format, from the host tables (CPU tensors)."""
        news = lambda row: {a: torch.tensor(t[row] if a in _LIST_FIELDS else t[row, 0], dtype=torch.int64)
                            for a, t in self.news_tables.items()}
        rows, rec = self.behaviors[idx], self.records[idx]
        item = {}
        if "user" in self.record_names:
            item["user"] = int(rec[0])
        item["clicked"] = [int(x) for x in rec[2:]]
        item["candidate_news"] = [news(r) for r in rows[self.H:]]
        if "clicked_news_length" in self.record_names:
            item["clicked_news_length"] = int(rec[1])
        item["clicked_news"] = [news(r) for r in rows[:self.H]]
        return item

    def loader(self, batch_size, shuffle=False, drop_last=False, *, rank=0, world=1, seed=0, epoch=0, **ignored):
        """The DataLoader stand-in: the reference's keyword arguments (num_workers, pin_memory are ignored)."""
        if self._dev is None:
            from . import NewsrecError
            raise NewsrecError("DeviceFeed.loader needs the tables on a CUDA device: the feed has no host path")
        if self.resample_negatives:
            self.draw(epoch)
        return FeedLoader(self, batch_size, shuffle, drop_last, rank, world, seed, epoch)


@dataclass
class ImpressionTables:
    """Host tables of a resampling feed (resample_tables); R = row_offsets[-1] rows."""
    behaviors: np.ndarray    # (R, H + 1 + K) int32: the history columns; the candidate columns are the draw's (zero here)
    records: np.ndarray      # (R, 3 + K) int32: user, clicked_news_length, then the labels 1, 0, ..., 0
    cand_rows: np.ndarray    # (n_cand,) int32 news rows, impressions back to back
    labels: np.ndarray       # (n_cand,) uint8, 1 positive / 0 negative
    imp_offsets: np.ndarray  # (n_imp + 1,) int64
    row_offsets: np.ndarray  # (n_imp + 1,) int64: impression i owns rows [row_offsets[i], row_offsets[i+1]), min(P, N // K) of them


def resample_tables(directory, news_index, H, K, user2int_path):
    """MIND's raw behaviors.tsv in `directory` as the tables of a resampling feed (no CUDA needed).  news_index maps news
    ids (and "PADDED_NEWS") to news rows; histories are the first H browsed news, left-padded with the padding news; users
    go through user2int.tsv.  Raises KeyError for an unknown news id, ValueError for a label other than 0 / 1 or a user
    user2int.tsv does not list."""
    import pandas as pd
    from .evaluate import impression_candidates, read_behaviors, user_tables
    beh = read_behaviors(directory)
    _, history, length, hist_row = user_tables(beh, news_index, H, user2int_path)
    user2int = dict(pd.read_table(user2int_path).values.tolist())
    users = beh["user"].tolist()
    unknown = sorted({u for u in users if u not in user2int})
    if unknown:
        raise ValueError(f"{directory}/behaviors.tsv: users not in {user2int_path}: {unknown[:5]}")
    hist = np.asarray([hist_row[h] for h in beh["clicked_news"].tolist()], np.int64)
    cand, labels, imp_offsets = impression_candidates(beh["impressions"], news_index)
    if ((labels != 0) & (labels != 1)).any():
        raise ValueError(f"{directory}/behaviors.tsv: a label other than 0 or 1 ({sorted(set(labels.tolist()) - {0, 1})[:5]})")
    counts = np.diff(imp_offsets)
    P = np.bincount(np.repeat(np.arange(len(counts)), counts), weights=labels, minlength=len(counts)).astype(np.int64)
    rows = np.minimum(P, (counts - P) // K)
    row_offsets = np.zeros(len(counts) + 1, np.int64)
    row_offsets[1:] = np.cumsum(rows)
    of_row = hist[np.repeat(np.arange(len(counts)), rows)]
    user = np.asarray([user2int[u] for u in users], np.int64)[np.repeat(np.arange(len(counts)), rows)]
    behaviors = np.zeros((len(of_row), H + 1 + K), np.int64)
    behaviors[:, :H] = history[of_row]
    records = np.zeros((len(of_row), 3 + K), np.int64)
    records[:, 0], records[:, 1], records[:, 2] = user, length[of_row], 1
    return ImpressionTables(behaviors=_int32(behaviors, "behaviour table"), records=_int32(records, "user column"),
                            cand_rows=_int32(cand, "news rows"), labels=labels.astype(np.uint8), imp_offsets=imp_offsets,
                            row_offsets=row_offsets)


def epoch_rows(n, batch_size, shuffle=False, drop_last=False, rank=0, world=1, seed=0, epoch=0):
    """The rows one rank visits in one epoch, batch after batch (host int64): a DistributedSampler over n rows, then the
    last incomplete batch dropped when drop_last is set."""
    from torch.utils.data.distributed import DistributedSampler
    sampler = DistributedSampler(range(n), num_replicas=world, rank=rank, shuffle=bool(shuffle), seed=seed, drop_last=bool(drop_last))
    sampler.set_epoch(epoch)
    order = torch.tensor(list(iter(sampler)), dtype=torch.int64)
    return order[:len(order) // batch_size * batch_size] if drop_last else order


class FeedLoader:
    """One epoch of batches; `len()` and `iter()` as a DataLoader's.  The row permutation is drawn on the host once per
    loader (DistributedSampler) and copied to the device once; each batch slices it."""

    def __init__(self, feed, batch_size, shuffle, drop_last, rank, world, seed, epoch):
        self.feed, self.B = feed, int(batch_size)
        order = epoch_rows(len(feed), self.B, shuffle, drop_last, rank, world, seed, epoch)
        self.rows = order.to(feed.device)
        self._n = -(-len(order) // self.B)

    def __len__(self):
        return self._n

    def __iter__(self):
        for i in range(self._n):
            with torch.cuda.device(self.feed.device):  # the library launches on the current device: make it the feed's
                batch = self._batch(self.rows[i * self.B:(i + 1) * self.B])
            yield batch

    def _batch(self, rows):
        from . import FeedField, check, load_library
        feed, dev = self.feed, self.feed.device
        B, H, Cn = rows.shape[0], feed.H, feed.C
        n = B * (H + Cn)
        blocks, fields = {}, []
        for a, t in feed._dev["news"].items():
            out = torch.empty((n, t.shape[1]) if a in _LIST_FIELDS else (n,), dtype=torch.int64, device=dev)
            blocks[a] = out
            fields.append(FeedField(t.data_ptr(), t.shape[1], out.data_ptr()))
        # user and clicked_news_length get buffers of their own: LSTUR's user encoder changes the lengths in place while
        # autograd holds the user ids (one storage would share one version counter)
        user = torch.empty(B, dtype=torch.int64, device=dev) if "user" in feed.record_names else None
        length = torch.empty(B, dtype=torch.int64, device=dev) if "clicked_news_length" in feed.record_names else None
        labels = torch.empty((Cn, B), dtype=torch.int64, device=dev)
        ptr = lambda t: C.c_void_p(t.data_ptr() if t is not None else None)
        table = (FeedField * max(1, len(fields)))(*fields)
        check(load_library().nr_feed_gather(table, len(fields), ptr(feed._dev["behaviors"]), H, Cn, ptr(feed._dev["records"]), ptr(rows), B,
                                            ptr(user), ptr(length), ptr(labels), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
              "nr_feed_gather")
        clicked = [dict() for _ in range(H)]
        cands = [dict() for _ in range(Cn)]
        for a, blk in blocks.items():
            tail = blk.shape[1:]
            for d, v in zip(clicked, blk[:B * H].view(B, H, *tail).unbind(1)):
                d[a] = v
            for d, v in zip(cands, blk[B * H:].view(B, Cn, *tail).unbind(1)):
                d[a] = v
        batch = {"candidate_news": FeedSlots(cands, blocks, B), "clicked_news": FeedSlots(clicked, blocks, B),
                 "clicked": list(labels.unbind(0))}
        if user is not None:
            batch["user"] = user
        if length is not None:
            batch["clicked_news_length"] = length
        return batch
