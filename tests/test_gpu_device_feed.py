"""Device feed on the H100: nr_feed_gather against NumPy, the blocks the models receive against SlotPacker.pack over the
reference-collated golden batch, one launch per batch and none in SlotPacker.pack, and a forward + backward of every family
on a feed batch against the same step on the collated CPU batch."""
import ctypes as C

import numpy as np
import pytest
import torch

import newsrec_b200
from feed_util import BEHAVIORS, FAMILIES, NEWS, family_config, golden, golden_arrays
from newsrec_b200 import FeedField, check, load_library
from newsrec_b200.feed import DeviceFeed, FeedSlots
from newsrec_b200.pack import SlotPacker

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
GUARD = 64
SENTINEL = -0x5A5A5A5A5A5A5A5


def _behaviour_table(rng, R, H, Cn, n_news, pad):
    """Rows whose histories are all padding, full, or truncated (left-padded) -- the three kinds the feed builds."""
    beh = rng.integers(0, n_news, size=(R, H + Cn), dtype=np.int64)
    for r in range(R):
        kind = r % 3
        if kind == 0:
            beh[r, :H] = pad
        elif kind == 2:
            beh[r, :rng.integers(0, H + 1)] = pad
    return beh.astype(np.int32)


def _guarded(n):
    buf = torch.full((n + 2 * GUARD,), SENTINEL, dtype=torch.int64, device=DEV)
    return buf, buf[GUARD:GUARD + n]


def _intact(buf, n, shift=0):
    host = buf.cpu().numpy()
    return (host[:GUARD + shift] == SENTINEL).all() and (host[GUARD + shift + n:] == SENTINEL).all()


def _run_gather(widths, B, Cn, H=50, R=700, n_news=300, records=True, offset_out=(), offset_table=None):
    rng = np.random.default_rng(B * 100 + Cn)
    tables = [rng.integers(0, 2 ** 31 - 1, size=(n_news + 1, w), dtype=np.int64).astype(np.int32) for w in widths]
    for t in tables:
        t[n_news] = 0
    beh = _behaviour_table(rng, R, H, Cn, n_news + 1, n_news)
    rec = rng.integers(-5, 1000, size=(R, 2 + Cn), dtype=np.int64).astype(np.int32)
    rows = rng.choice(R, size=B, replace=B > R).astype(np.int64)
    d = lambda a: torch.from_numpy(a).to(DEV)
    n = B * (H + Cn)
    outs, views, fields = [], [], []
    for f, w in enumerate(widths):
        shift = 1 if f in offset_out else 0  # 8 bytes off 16-byte alignment: the scalar path
        buf = torch.full((n * w + 2 * GUARD + shift,), SENTINEL, dtype=torch.int64, device=DEV)
        outs.append(buf)
        views.append(buf[GUARD + shift:GUARD + shift + n * w].view(n, w))
    dt = []
    for f, t in enumerate(tables):
        shift = (offset_table or {}).get(f, 0)  # int32 elements off the allocation's 16-byte alignment
        flat = torch.zeros(t.size + shift, dtype=torch.int32, device=DEV)
        flat[shift:] = d(t.reshape(-1))
        dt.append(flat[shift:].view(t.shape))
    for t, v in zip(dt, views):
        fields.append(FeedField(t.data_ptr(), t.shape[1], v.data_ptr()))
    (ub, u), (lb, ln), (cb, cl) = _guarded(B), _guarded(B), _guarded(Cn * B)
    d_beh, d_rec, d_rows = d(beh), d(rec), d(rows)
    ptr = lambda t: C.c_void_p(t.data_ptr() if records else None)
    table = (FeedField * len(fields))(*fields)
    before = newsrec_b200.launch_count()
    check(load_library().nr_feed_gather(table, len(fields), C.c_void_p(d_beh.data_ptr()), H, Cn, ptr(d_rec), C.c_void_p(d_rows.data_ptr()),
                                        B, ptr(u), ptr(ln), ptr(cl), C.c_void_p(torch.cuda.current_stream().cuda_stream)), "nr_feed_gather")
    torch.cuda.synchronize()
    assert newsrec_b200.launch_count() == before + 1
    order = np.concatenate([beh[rows, :H].reshape(-1), beh[rows, H:].reshape(-1)])  # impression-major browsed, then candidates
    for f, (t, buf, v) in enumerate(zip(tables, outs, views)):
        np.testing.assert_array_equal(v.cpu().numpy(), t[order].astype(np.int64), err_msg=f"field {f} width {widths[f]}")
        assert _intact(buf, n * widths[f], 1 if f in offset_out else 0)
    if records:
        np.testing.assert_array_equal(u.cpu().numpy(), rec[rows, 0].astype(np.int64))
        np.testing.assert_array_equal(ln.cpu().numpy(), rec[rows, 1].astype(np.int64))
        np.testing.assert_array_equal(cl.view(Cn, B).cpu().numpy(), rec[rows, 2:].T.astype(np.int64))
    else:
        assert (u.cpu() == SENTINEL).all() and (ln.cpu() == SENTINEL).all() and (cl.cpu() == SENTINEL).all()
    assert _intact(ub, B) and _intact(lb, B) and _intact(cb, Cn * B)


@pytest.mark.parametrize("B", [1, 3, 512])
@pytest.mark.parametrize("Cn", [3, 5])
def test_gather_equals_numpy(B, Cn):
    _run_gather((1, 20, 50), B, Cn)


def test_gather_unaligned_output_and_no_history():
    _run_gather((20, 50, 1), 37, 5, offset_out=(0, 1))  # 16-byte stores impossible: the scalar path
    _run_gather((20,), 9, 4, H=0, records=False)
    # tables off alignment: 8 bytes (width 20: 8-byte loads, 16-byte stores) and 4 bytes (the scalar path)
    _run_gather((20, 20, 50), 37, 5, offset_table={0: 2, 1: 1, 2: 1})


@pytest.mark.parametrize("drop_last", [False, True])
def test_loader_iterates_the_epoch_rows_batch_by_batch(drop_last):
    """A shuffled loader over the 12 golden rows in batches of 5: every batch holds the rows epoch_rows gives for its
    position (the short last batch too unless drop_last), each field block is the host tables' gather of those rows."""
    from newsrec_b200.feed import epoch_rows
    cfg = family_config("LSTUR")
    feed = DeviceFeed(BEHAVIORS, NEWS, cfg, device=DEV)
    H, Cn, R = feed.H, feed.C, len(feed)
    orders = []
    for epoch in (0, 1):
        rows = epoch_rows(R, 5, shuffle=True, drop_last=drop_last, seed=4, epoch=epoch).numpy()
        orders.append(rows.tolist())
        loader = feed.loader(5, shuffle=True, drop_last=drop_last, seed=4, epoch=epoch, num_workers=4, pin_memory=True)
        sizes = [5, 5] if drop_last else [5, 5, 2]
        assert len(loader) == len(sizes)
        seen = 0
        for i, batch in enumerate(loader):
            r = rows[seen:seen + sizes[i]]
            seen += sizes[i]
            rec = feed.records[r].astype(np.int64)
            assert batch["user"].shape == (len(r),)
            np.testing.assert_array_equal(batch["user"].cpu().numpy(), rec[:, 0])
            np.testing.assert_array_equal(batch["clicked_news_length"].cpu().numpy(), rec[:, 1])
            np.testing.assert_array_equal(torch.stack(batch["clicked"]).cpu().numpy(), rec[:, 2:].T)
            beh = feed.behaviors[r]
            news_rows = np.concatenate([beh[:, :H].reshape(-1), beh[:, H:].reshape(-1)])
            for attr, table in feed.news_tables.items():
                got = batch["clicked_news"].blocks[attr].cpu().numpy().reshape(len(news_rows), -1)
                np.testing.assert_array_equal(got, table[news_rows].astype(np.int64), err_msg=attr)
        assert i + 1 == len(sizes) and seen == len(rows)
    assert orders[0] != orders[1]  # a re-created loader (next epoch) draws a new permutation


def test_gather_refuses_bad_arguments():
    lib = load_library()
    before = newsrec_b200.launch_count()
    f = (FeedField * 9)()
    p = C.c_void_p(16)
    assert lib.nr_feed_gather(f, 9, p, 50, 5, None, p, 4, None, None, None, None) == -1  # more than 8 fields
    assert lib.nr_feed_gather(f, 1, p, 50, 5, None, p, 4, None, None, None, None) == -1  # null table
    assert lib.nr_feed_gather(f, 0, p, 50, 0, None, p, 4, None, None, None, None) == -1  # C = 0
    assert lib.nr_feed_gather(f, 0, p, 50, 5, None, p, 4, p, None, None, None) == -1     # an output without the records
    assert newsrec_b200.launch_count() == before


def _feed_batch(fam, cfg=None):
    """The golden rows, in the golden order, as one batch of the device feed."""
    g = golden()
    cfg = cfg or family_config(fam)
    feed = DeviceFeed(BEHAVIORS, NEWS, cfg, device=DEV)
    order = g[f"{fam}.order"]
    loader = feed.loader(len(order), shuffle=False, drop_last=True)
    loader.rows = torch.from_numpy(order).to(DEV)
    it = iter(loader)
    before = newsrec_b200.launch_count()
    batch = next(it)
    assert newsrec_b200.launch_count() == before + 1  # one gather per batch
    with pytest.raises(StopIteration):
        next(it)
    return batch, g, cfg


def _cpu_batch(g, fam, cfg):
    """The reference-collated batch as the trainer receives it from the reference's DataLoader (CPU tensors)."""
    a = golden_arrays(g, fam)
    mk = lambda key, n: [{attr: torch.from_numpy(a[f"{key}.{attr}"][s]).contiguous() for attr in cfg.dataset_attributes["news"]}
                         for s in range(n)]
    batch = {"clicked_news": mk("clicked_news", cfg.num_clicked_news_a_user), "candidate_news": mk("candidate_news", a["clicked"].shape[0]),
             "clicked": [torch.from_numpy(x) for x in a["clicked"]]}
    for rec in cfg.dataset_attributes["record"]:
        batch[rec] = torch.from_numpy(a[rec])
    return batch


@pytest.mark.parametrize("fam", FAMILIES)
def test_feed_blocks_equal_slot_packer_over_the_golden_batch(fam):
    batch, g, cfg = _feed_batch(fam)
    cpu = _cpu_batch(g, fam, cfg)
    assert isinstance(batch["clicked_news"], FeedSlots) and isinstance(batch["candidate_news"], FeedSlots)
    # the slot views hold the reference loader's values
    for key in ("clicked_news", "candidate_news"):
        assert len(batch[key]) == len(cpu[key])
        for got, want in zip(batch[key], cpu[key]):
            assert sorted(got) == sorted(want)
            for attr in want:
                assert got[attr].device == DEV and torch.equal(got[attr].cpu(), want[attr]), (key, attr)
    for k in ["clicked"]:
        assert all(torch.equal(x.cpu(), y) for x, y in zip(batch[k], cpu[k]))
    for rec in ("user", "clicked_news_length"):
        assert (rec in batch) == (rec in cfg.dataset_attributes["record"])
        if rec in batch:
            assert batch[rec].dtype == torch.int64 and torch.equal(batch[rec].cpu(), cpu[rec])
    packer, ref = SlotPacker(), SlotPacker()
    for attr in cfg.dataset_attributes["news"]:
        before = newsrec_b200.launch_count()
        ids, B = packer.pack(batch["clicked_news"], batch["candidate_news"], attr, DEV)
        assert newsrec_b200.launch_count() == before  # the block is handed over, nothing launched
        want, B_ref = ref.pack(cpu["clicked_news"], cpu["candidate_news"], attr, DEV)
        assert B == B_ref and ids.dtype == want.dtype and torch.equal(ids, want), attr


# Bit-identical logits for every family.  Gradients: a family whose backward gives the same bits in three runs on the
# collated batch must give those bits on the feed batch too.  Where floating-point atomics (additive-attention and
# weight-gradient reductions, embedding scatters) make runs differ in the last bits -- on the H100 that is every family here:
# NRMS, NAML, LSTUR, TANR, Exp1, Hi-Fi Ark and DKN -- each gradient's difference from the feed batch must stay within 4x the
# largest relative difference between those three runs.  The bound is per family, not per gradient: an analytically zero
# gradient (the key bias of a self-attention) can agree in three runs by chance and still differ in a fourth.
RUNS = 3


def _model(fam, cfg):
    import importlib
    torch.manual_seed(1234)
    Model = getattr(importlib.import_module("model." + fam), fam)
    return Model(cfg).to(DEV).train()


def _step(model, fam, batch):
    torch.manual_seed(99)
    model.zero_grad(set_to_none=True)
    args = (batch["candidate_news"], batch["clicked_news"])
    out = model(batch["user"], batch["clicked_news_length"], *args) if fam == "LSTUR" else model(*args)
    logits, aux = out if isinstance(out, tuple) else (out, None)
    loss = torch.nn.functional.cross_entropy(logits, torch.zeros(logits.shape[0], dtype=torch.long, device=DEV))
    if aux is not None:
        loss = loss + 0.1 * aux
    loss.backward()
    torch.cuda.synchronize()
    return logits.detach().clone(), {k: p.grad.detach().clone() for k, p in model.named_parameters() if p.grad is not None}


@pytest.mark.parametrize("fam", FAMILIES)
def test_family_step_on_a_feed_batch_equals_the_collated_batch(fam):
    cfg = family_config(fam, num_words=1000, num_categories=64, num_users=50, num_entities=500, dropout_probability=0.0,
                        masking_probability=0.0)
    model = _model(fam, cfg)
    batch, g, _ = _feed_batch(fam, cfg)
    cpu = _cpu_batch(g, fam, cfg)
    newsrec_b200.load_library().nr_profile_enable(1)
    newsrec_b200.profile_report()
    try:
        logits_f, grads_f = _step(model, fam, batch)
        launched = newsrec_b200.profile_report()
    finally:
        newsrec_b200.load_library().nr_profile_enable(0)
    assert not any("pack_slots" in k for k in launched), sorted(launched)
    runs = [_step(model, fam, cpu) for _ in range(RUNS)]
    logits_c, grads_c = runs[0]
    for lg, _ in runs:
        assert torch.equal(logits_f, lg)
    assert sorted(grads_f) == sorted(grads_c) and grads_f
    rel = lambda a, b: float((a - b).norm() / b.norm().clamp_min(1e-30))
    spread = max(rel(gr[k], grads_c[k]) for _, gr in runs[1:] for k in grads_c)
    if spread == 0.0:
        for k in grads_c:
            assert torch.equal(grads_f[k], grads_c[k]), k
    else:
        assert spread < 1e-4, spread  # run-to-run noise of atomics, not a different computation
        for k in grads_c:
            assert rel(grads_f[k], grads_c[k]) <= 4 * spread, (k, rel(grads_f[k], grads_c[k]), spread)
