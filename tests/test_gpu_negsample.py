"""Training negatives on the H100: nr_sample_negatives bit for bit against the NumPy oracle (oracle/negsample_oracle.py)
with sentinel guards, its statistics over many epochs, the resampling DeviceFeed against a plain DeviceFeed over the
oracle's draw written as behaviors_parsed.tsv, launch counts, two ranks, a training step of NRMS and LSTUR, and the
refused arguments."""
import ctypes as C
import os

import numpy as np
import pytest
import torch
from scipy import stats

import newsrec_b200
from feed_util import ROOT, family_config
from negsample_oracle import draw
from newsrec_b200 import load_library
from newsrec_b200.feed import DeviceFeed, epoch_rows

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
SENTINEL = -0x5A5A5A5
GUARD_ROWS = 3
FIXTURE = os.path.join(ROOT, "tests", "golden", "negsample")
ptr = lambda t: C.c_void_p(t.data_ptr())


def _impressions(rng, sizes):
    """CSR of impressions with (P, N) = sizes, labels in random order, news rows < 10^6."""
    cand, labels, offsets = [], [], [0]
    for P, N in sizes:
        lab = np.array([1] * P + [0] * N, np.uint8)
        rng.shuffle(lab)
        labels.append(lab)
        cand.append(rng.integers(0, 10 ** 6, size=P + N))
        offsets.append(offsets[-1] + P + N)
    cat = lambda xs, dt: np.concatenate(xs).astype(dt) if xs else np.zeros(0, dt)
    return cat(cand, np.int32), cat(labels, np.uint8), np.asarray(offsets, np.int64)


def _run(cand, labels, offsets, K, seed, epoch, H=5, table=None):
    """Launch the draw into a sentinel-filled table with GUARD_ROWS guard rows on each side; returns (table, owned view)."""
    from negsample_oracle import balanced_rows
    rows = balanced_rows(labels, offsets, K)
    row_offsets = np.concatenate([[0], np.cumsum(rows)]).astype(np.int64)
    R, W = int(row_offsets[-1]), H + 1 + K
    if table is None:
        table = torch.full((R + 2 * GUARD_ROWS, W), SENTINEL, dtype=torch.int32, device=DEV)
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    dc, dl, do, dr = d(cand), d(labels), d(offsets), d(row_offsets)
    before = newsrec_b200.launch_count()
    rc = load_library().nr_sample_negatives(ptr(dc), ptr(dl), ptr(do), len(offsets) - 1, ptr(dr), K, seed & (2 ** 64 - 1), epoch,
                                            ptr(table[GUARD_ROWS:]), H, C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0, load_library().nr_last_error()
    torch.cuda.synchronize()
    assert newsrec_b200.launch_count() == before + (1 if len(offsets) > 1 else 0)
    return table, row_offsets


def _check(cand, labels, offsets, K, seed, epoch, H=5):
    table, row_offsets = _run(cand, labels, offsets, K, seed, epoch, H)
    host = table.cpu().numpy()
    R = int(row_offsets[-1])
    want_offsets, want = draw(cand, labels, offsets, K, seed, epoch)
    np.testing.assert_array_equal(row_offsets, want_offsets)
    np.testing.assert_array_equal(host[GUARD_ROWS:GUARD_ROWS + R, H:], want, err_msg=f"K={K} seed={seed} epoch={epoch}")
    assert (host[GUARD_ROWS:GUARD_ROWS + R, :H] == SENTINEL).all()  # history columns untouched
    assert (host[:GUARD_ROWS] == SENTINEL).all() and (host[GUARD_ROWS + R:] == SENTINEL).all()  # guard rows untouched
    return host


@pytest.mark.parametrize("K", [1, 2, 4])
def test_draw_equals_the_oracle(K):
    rng = np.random.default_rng(K)
    sizes = [(int(rng.integers(0, 11)), int(n)) for n in rng.integers(0, 80, size=300)]
    sizes += [(0, 0), (3, 0), (0, 9), (1, K - 1), (10, 3 * K), (2, 255), (4, 256), (5, 257), (10, 1000), (7, 4100), (1, 4097)]
    rng.shuffle(sizes)
    cand, labels, offsets = _impressions(rng, sizes)
    for seed, epoch in [(0, 0), (0, 1), (123456789, 7), (2 ** 64 - 1, 2 ** 40 + 3), (42, -1)]:
        _check(cand, labels, offsets, K, seed, epoch)


def test_draw_without_history_and_with_one_impression():
    rng = np.random.default_rng(9)
    cand, labels, offsets = _impressions(rng, [(2, 9)])
    _check(cand, labels, offsets, 4, 5, 0, H=0)
    cand, labels, offsets = _impressions(rng, [(3, 6000)])  # one long impression, staged tile by tile
    _check(cand, labels, offsets, 2, 5, 3, H=2)


def test_inclusion_rates_and_epoch_overlap():
    """Over 400 epochs every negative of an impression is picked equally often (chi-square), and the picks of consecutive
    epochs overlap as drawing M of N without replacement twice, independently, predicts (hypergeometric)."""
    N, P, K, E = 24, 3, 2, 400
    M = P * K
    rng = np.random.default_rng(11)
    cand, labels, offsets = _impressions(rng, [(P, N)] * 64)
    cand = np.arange(len(cand), dtype=np.int32)  # a candidate's row is its position: picks identify negatives
    counts = np.zeros(len(cand), np.int64)
    prev, overlaps = None, []
    for e in range(E):
        table, row_offsets = _run(cand, labels, offsets, K, 77, e, H=1)
        picks = table[GUARD_ROWS:GUARD_ROWS + int(row_offsets[-1]), 2:].cpu().numpy().reshape(64, M)
        np.add.at(counts, picks.reshape(-1), 1)
        if prev is not None:
            overlaps += [len(set(a) & set(b)) for a, b in zip(prev, picks)]
        prev = picks
    neg = labels == 0
    assert counts[~neg].sum() == 0
    for i in range(64):
        c = counts[offsets[i]:offsets[i + 1]][neg[offsets[i]:offsets[i + 1]]]
        assert c.sum() == E * M
        assert stats.chisquare(c).pvalue > 1e-4, (i, c)
    obs = np.bincount(overlaps, minlength=M + 1)
    pmf = stats.hypergeom(N, M, M).pmf(np.arange(M + 1))
    keep = pmf * len(overlaps) >= 5  # pool the sparse tails
    f_obs = np.append(obs[keep], obs[~keep].sum())
    f_exp = np.append(pmf[keep], pmf[~keep].sum()) * len(overlaps)
    assert stats.chisquare(f_obs, f_exp).pvalue > 1e-4, (obs, pmf * len(overlaps))


def test_refused_arguments_launch_nothing():
    lib = load_library()
    p = C.c_void_p(256)
    before = newsrec_b200.launch_count()
    assert lib.nr_sample_negatives(None, p, p, 1, p, 2, 0, 0, p, 5, None) == -1
    assert lib.nr_sample_negatives(p, None, p, 1, p, 2, 0, 0, p, 5, None) == -1
    assert lib.nr_sample_negatives(p, p, None, 1, p, 2, 0, 0, p, 5, None) == -1
    assert lib.nr_sample_negatives(p, p, p, 1, None, 2, 0, 0, p, 5, None) == -1
    assert lib.nr_sample_negatives(p, p, p, 1, p, 2, 0, 0, None, 5, None) == -1
    assert lib.nr_sample_negatives(p, p, p, 1, p, 0, 0, 0, p, 5, None) == -1   # K < 1
    assert lib.nr_sample_negatives(p, p, p, -1, p, 2, 0, 0, p, 5, None) == -1  # n_imp < 0
    assert lib.nr_sample_negatives(p, p, p, 1, p, 2, 0, 0, p, -1, None) == -1  # H < 0
    assert b"nr_sample_negatives" in lib.nr_last_error()
    assert lib.nr_sample_negatives(p, p, p, 0, p, 2, 0, 0, p, 5, None) == 0    # no impression: nothing to do
    assert newsrec_b200.launch_count() == before


# ---- the resampling feed --------------------------------------------------------------------------------------------------

def _feed(cfg=None, seed=3):
    cfg = cfg or family_config("LSTUR")
    return DeviceFeed(os.path.join(FIXTURE, "behaviors_parsed.tsv"), os.path.join(FIXTURE, "news_parsed.tsv"), cfg, device=DEV,
                      resample_negatives=True, seed=seed)


def _plain_feed_of_the_oracle(tmp_path, feed, epoch):
    """behaviors_parsed.tsv written from the oracle's draw of `epoch`, and a plain DeviceFeed over it."""
    from newsrec_b200.evaluate import read_behaviors, read_news
    ids, _ = read_news(FIXTURE, ["title"])
    t = feed.impressions
    row_offsets, cand = draw(t.cand_rows, t.labels, t.imp_offsets, feed.K, feed.seed, epoch)
    beh = read_behaviors(FIXTURE)
    imp = np.repeat(np.arange(len(beh)), np.diff(row_offsets))
    path = tmp_path / f"behaviors_parsed_{epoch}.tsv"
    with open(path, "w") as f:
        f.write("user\tclicked_news\tcandidate_news\tclicked\n")
        for r, i in enumerate(imp):
            f.write(f"{t.records[r, 0]}\t{beh['clicked_news'][i]}\t{' '.join(ids[x] for x in cand[r])}\t{' '.join(['1'] + ['0'] * feed.K)}\n")
    return DeviceFeed(str(path), os.path.join(FIXTURE, "news_parsed.tsv"), feed.config, device=DEV)


def _batches(loader):
    out = []
    for b in loader:
        blocks = {a: v.cpu().numpy() for a, v in b["clicked_news"].blocks.items()}
        out.append((blocks, b["user"].cpu().numpy(), b["clicked_news_length"].cpu().numpy(), torch.stack(b["clicked"]).cpu().numpy()))
    return out


def test_feed_batches_equal_a_plain_feed_over_the_oracle_draw(tmp_path):
    feed = _feed()
    n = len(feed)
    for epoch in (0, 1, 2, 5):
        plain = _plain_feed_of_the_oracle(tmp_path, feed, epoch)
        got = _batches(feed.loader(4, shuffle=True, drop_last=False, seed=8, epoch=epoch))
        want = _batches(plain.loader(4, shuffle=True, drop_last=False, seed=8, epoch=epoch))
        assert len(feed) == len(plain) == n  # the same length every epoch
        assert len(got) == len(want)
        for (gb, *gr), (wb, *wr) in zip(got, want):
            assert sorted(gb) == sorted(wb)
            for a in wb:
                np.testing.assert_array_equal(gb[a], wb[a], err_msg=(epoch, a))
            for x, y in zip(gr, wr):
                np.testing.assert_array_equal(x, y)
        np.testing.assert_array_equal(feed.behaviors, plain.behaviors)
        np.testing.assert_array_equal(feed.records, plain.records)
        for idx in (0, n // 2, n - 1):  # feed[idx] is the current epoch's row
            a, b = feed[idx], plain[idx]
            assert a["clicked"] == b["clicked"] and a["user"] == b["user"] and a["clicked_news_length"] == b["clicked_news_length"]
            for key in ("candidate_news", "clicked_news"):
                for x, y in zip(a[key], b[key]):
                    assert all(torch.equal(x[k], y[k]) for k in y)


def test_one_launch_per_draw_and_one_per_batch():
    feed = _feed()
    before = newsrec_b200.launch_count()
    loader = feed.loader(5, shuffle=True, epoch=0)  # construction drew epoch 0 already
    assert newsrec_b200.launch_count() == before
    for _ in loader:
        pass
    assert newsrec_b200.launch_count() == before + len(loader)
    before = newsrec_b200.launch_count()
    loader = feed.loader(5, shuffle=True, epoch=1)
    assert newsrec_b200.launch_count() == before + 1
    for _ in loader:
        pass
    assert newsrec_b200.launch_count() == before + 1 + len(loader)
    before = newsrec_b200.launch_count()
    feed.loader(5, shuffle=True, epoch=1)
    assert newsrec_b200.launch_count() == before


def test_two_ranks_hold_the_same_table_and_disjoint_rows():
    f0, f1 = _feed(seed=21), _feed(seed=21)
    for epoch in (0, 3):
        l0 = f0.loader(3, shuffle=True, drop_last=True, rank=0, world=2, seed=21, epoch=epoch)
        l1 = f1.loader(3, shuffle=True, drop_last=True, rank=1, world=2, seed=21, epoch=epoch)
        assert torch.equal(f0._dev["behaviors"], f1._dev["behaviors"])
        r0, r1 = set(l0.rows.cpu().tolist()), set(l1.rows.cpu().tolist())
        assert r0 and r1 and not r0 & r1
        assert l0.rows.cpu().tolist() == epoch_rows(len(f0), 3, True, True, 0, 2, 21, epoch).tolist()
    assert not torch.equal(f0._dev["behaviors"], _feed(seed=22)._dev["behaviors"])


@pytest.mark.parametrize("fam", ["NRMS", "LSTUR"])
def test_training_step_on_resampled_batches(fam):
    import importlib
    cfg = family_config(fam, num_words=1000, num_categories=64, num_users=50, num_entities=500, dropout_probability=0.0,
                        masking_probability=0.0)
    torch.manual_seed(1234)
    model = getattr(importlib.import_module("model." + fam), fam)(cfg).to(DEV).train()
    feed = _feed(cfg)
    for epoch in (0, 1):
        for batch in feed.loader(8, shuffle=True, epoch=epoch):
            model.zero_grad(set_to_none=True)
            args = (batch["candidate_news"], batch["clicked_news"])
            out = model(batch["user"], batch["clicked_news_length"], *args) if fam == "LSTUR" else model(*args)
            logits = out[0] if isinstance(out, tuple) else out
            assert logits.shape == (batch["clicked"][0].shape[0], 1 + cfg.negative_sampling_ratio)
            loss = torch.nn.functional.cross_entropy(logits, torch.zeros(logits.shape[0], dtype=torch.long, device=DEV))
            loss.backward()
            assert torch.isfinite(loss)
            grads = [p.grad for p in model.parameters() if p.grad is not None]
            assert grads and all(torch.isfinite(g).all() for g in grads)
