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
"""
from __future__ import annotations

import ctypes as C
import os

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
    `news_tables`, `behaviors`, `records`) and copied to `device` (default: the current CUDA device, if any)."""

    def __init__(self, behaviors_path, news_path, config=None, device=None):
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

        beh = pd.read_table(behaviors_path)
        R = len(beh)
        C = None
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
        self.behaviors = _int32(np.asarray(behaviors, np.int64).reshape(R, H + C), "behaviour table")
        self.records = _int32(np.asarray(records, np.int64).reshape(R, 2 + C), "user / clicked columns")

        if device is None and torch.cuda.is_available():
            device = torch.device("cuda", torch.cuda.current_device())
        self.device = torch.device(device) if device is not None else None
        if self.device is not None and self.device.type == "cuda" and self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self._dev = None
        if self.device is not None and self.device.type == "cuda":
            to = lambda a: torch.from_numpy(a).to(self.device)
            self._dev = {"news": {a: to(t) for a, t in self.news_tables.items()}, "behaviors": to(self.behaviors),
                         "records": to(self.records)}

    def __len__(self):
        return len(self.behaviors)

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
        return FeedLoader(self, batch_size, shuffle, drop_last, rank, world, seed, epoch)


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
