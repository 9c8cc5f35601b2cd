"""Time windows over the news pool: recommend and rank only the news live at each request's time.

MIND news lives for a day or two, and ``news_parsed.tsv`` holds every news of a split's weeks, so a request should only see
the news shown around its own time.  This module owns that policy; the kernels only see one news-row range per request
(``ops.top_k_scores(..., row_range=)``, ``ops.pool_ranks(..., row_range=)``).

- **Time of a behaviors row.**  MIND's ``%m/%d/%Y %I:%M:%S %p`` (``11/15/2019 8:55:22 AM``) as int64 seconds, naive time
  (no zone).  A time that does not parse raises NewsrecError.
- **first_shown(n).**  The earliest time of a row of the split's ``behaviors.tsv`` whose impressions list news id n,
  labelled or not; history mentions do not count.  MIND has no publish times, so first appearance is the proxy.  Every pool
  row of an id gets the id's value; a news never listed has none and is in no window.
- **Eligible pool.**  For a request at time t and W = max_age_hours * 3600 seconds (a real number > 0; inf means every news
  shown so far), the news n with t - W <= first_shown(n) <= t, both ends inclusive, minus the request's exclusions.
- **Time order.**  The pool sorted once, stably, by (first_shown, news_parsed row) with the never-shown news first
  (``perm``: time-order position -> pool row; ``inv``: pool row -> position).  Each request's eligible news is then one
  contiguous range [lo, hi) of the time order (``PoolWindow.ranges``, two searchsorted calls).

A windowed call does all its device work in time order: the pool matrix is permuted once (one gather), categories through
``perm``, exclusions and targets through ``inv``, and the returned rows go back through ``perm`` once at the end (-1 kept).
The one visible consequence: among exactly equal scores, the news that comes first is the one earlier in time order rather
than the lower ``news_parsed`` row.
"""
from __future__ import annotations

import numbers
import os

import numpy as np

from . import NewsrecError

TIME_FORMAT = "%m/%d/%Y %I:%M:%S %p"


def max_age_seconds(who, max_age_hours):
    """W in seconds for max_age_hours (a real number > 0, inf allowed); raises NewsrecError on anything else (NaN, bools,
    strings, zero and negative values)."""
    if isinstance(max_age_hours, bool) or not isinstance(max_age_hours, numbers.Real) or not float(max_age_hours) > 0.0:
        raise NewsrecError(f"{who}: max_age_hours={max_age_hours!r} must be a real number > 0 (inf: no age limit)")
    return float(max_age_hours) * 3600.0


def parse_times(values, who="window"):
    """int64 seconds since 1970-01-01 00:00:00 (naive time) of MIND times ``%m/%d/%Y %I:%M:%S %p``; raises NewsrecError on
    a value that does not parse, an empty one included."""
    import pandas as pd
    s = pd.Series(list(values), dtype=object)
    try:
        t = pd.to_datetime(s, format=TIME_FORMAT)
    except (ValueError, TypeError) as e:
        raise NewsrecError(f"{who}: a behaviors.tsv time is not of the form {TIME_FORMAT!r}: {e}") from None
    if t.isna().any():
        raise NewsrecError(f"{who}: behaviors.tsv row {int(np.flatnonzero(t.isna().to_numpy())[0])} has no time")
    return t.to_numpy().astype("datetime64[s]").astype(np.int64)


def first_shown(beh, times, news_ids):
    """(first, shown) over the pool rows with ids news_ids: first (n,) int64 the earliest times[i] of a row i of beh
    (evaluate.read_behaviors) whose impressions list the row's id, shown (n,) bool whether there is one (first is 0 where
    not)."""
    import pandas as pd
    items = beh["impressions"].fillna("").astype(str).reset_index(drop=True).str.split().explode().dropna()
    ids = items.str.partition("-")[0].to_numpy(dtype=object) if len(items) else np.zeros(0, dtype=object)
    at = np.asarray(times, np.int64)[items.index.to_numpy(np.int64)]
    earliest = pd.Series(at, index=ids).groupby(level=0).min()
    got = earliest.reindex(pd.Index(news_ids, dtype=object))
    shown = got.notna().to_numpy()
    return np.where(shown, got.fillna(0).to_numpy(), 0).astype(np.int64), shown


class PoolWindow:
    """The time order of a pool (module docstring): perm, inv and the request ranges."""

    def __init__(self, first, shown):
        first, shown = np.asarray(first, np.int64), np.asarray(shown, bool)
        self.first, self.shown = first, shown
        self.perm = np.argsort(np.where(shown, first, np.iinfo(np.int64).min), kind="stable").astype(np.int64)
        self.inv = np.empty_like(self.perm)
        self.inv[self.perm] = np.arange(len(self.perm), dtype=np.int64)
        self.n_never = int(np.count_nonzero(~shown))
        self._sorted = first[self.perm[self.n_never:]].astype(np.float64)  # exact: |seconds| < 2^53

    def ranges(self, t, W):
        """(lo, hi) int64 arrays: the time-order positions [lo, hi) of the news with t - W <= first_shown <= t, per request
        time t (int64 seconds), W seconds (> 0, inf allowed)."""
        t = np.asarray(t, np.int64).astype(np.float64)
        lo = self.n_never + np.searchsorted(self._sorted, np.ceil(t - W), side="left")
        hi = self.n_never + np.searchsorted(self._sorted, t, side="right")
        return lo.astype(np.int64), hi.astype(np.int64)

    def to_time_order(self, rows):
        """Pool rows -> time-order positions (host int64 array; negative entries kept as they are)."""
        rows = np.asarray(rows, np.int64)
        return np.where(rows >= 0, self.inv[np.maximum(rows, 0)], rows)

    def to_rows(self, idx):
        """Time-order positions -> pool rows for a device or host int64 tensor / array; -1 (and any negative) kept."""
        if isinstance(idx, np.ndarray):
            return np.where(idx >= 0, self.perm[np.maximum(idx, 0)], idx)
        import torch
        perm = torch.from_numpy(self.perm).to(idx.device)
        return torch.where(idx >= 0, perm[idx.clamp(min=0)], idx)


def load(who, directory, max_age_hours):
    """Everything a windowed call checks before any device work: (W seconds, the read behaviors.tsv, its times), or None
    without max_age_hours.  Raises NewsrecError on a bad max_age_hours or a time that does not parse."""
    if max_age_hours is None:
        return None
    from .evaluate import read_behaviors
    W = max_age_seconds(who, max_age_hours)
    if not os.path.isfile(os.path.join(directory, "behaviors.tsv")):
        raise FileNotFoundError(f"{who}: {os.path.join(directory, 'behaviors.tsv')} not found")
    beh = read_behaviors(directory)
    return W, beh, parse_times(beh["time"].tolist(), who)


def pool_window(beh, times, news_ids):
    """The PoolWindow of the pool rows with ids news_ids under the impressions of beh."""
    return PoolWindow(*first_shown(beh, times, news_ids))


def csr_take(offsets, order):
    """Reorder the segments of a CSR: (gather, new_offsets) with segment j of the result segment order[j] of offsets, its
    entries at gather (entry i of the result is entry gather[i] of the input)."""
    offsets = np.asarray(offsets, np.int64)
    counts = np.diff(offsets)[order]
    new_offsets = np.zeros(len(order) + 1, np.int64)
    new_offsets[1:] = np.cumsum(counts)
    gather = np.repeat(offsets[:-1][order] - new_offsets[:-1], counts) + np.arange(new_offsets[-1], dtype=np.int64)
    return gather, new_offsets
