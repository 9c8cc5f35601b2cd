"""Host-side logic on CPU: the drop-in surface (class / method / state_dict names, config knobs), batch packing,
operand caching, the data-parallel plumbing over gloo (world_size 2), and 'no silent CPU fallback'."""
import os
import sys

import pytest
import torch

import newsrec_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

REFERENCE_DEFAULTS = dict(  # reference src/config.py:14-39 (BaseConfig) and :42-95
    num_epochs=2, num_batches_show_loss=100, num_batches_validate=1000, batch_size=128, learning_rate=0.0001, num_workers=4,
    num_clicked_news_a_user=50, num_words_title=20, num_words_abstract=50, word_freq_threshold=1, entity_freq_threshold=2,
    entity_confidence_threshold=0.5, negative_sampling_ratio=2, dropout_probability=0.2, num_words=70976, num_categories=275,
    num_entities=12958, num_users=50001, word_embedding_dim=300, category_embedding_dim=100, entity_embedding_dim=100,
    query_vector_dim=200)


def test_config_mirror_exposes_the_reference_knobs():
    import config
    assert config.model_name in ("NRMS", "NAML", "LSTUR", "TANR")
    for k, v in REFERENCE_DEFAULTS.items():
        assert getattr(config.BaseConfig, k) == v, k
    assert config.NRMSConfig.num_attention_heads == 15 and config.NRMSConfig.dataset_attributes == {"news": ["title"], "record": []}
    assert config.NAMLConfig.num_filters == 300 and config.NAMLConfig.window_size == 3
    assert config.NAMLConfig.dataset_attributes["news"] == ["category", "subcategory", "title", "abstract"]
    assert config.LSTURConfig.long_short_term_method == "ini" and config.LSTURConfig.masking_probability == 0.5
    assert config.LSTURConfig.dataset_attributes["record"] == ["user", "clicked_news_length"]
    assert config.TANRConfig.topic_classification_loss_weight == 0.1


@pytest.mark.parametrize("name,shapes", [("NRMS", lambda: O.nrms_shapes(70976)), ("NAML", lambda: O.naml_shapes(70976, 275)),
                                         ("TANR", lambda: O.tanr_shapes(70976, 275)), ("LSTUR", lambda: O.lstur_shapes(70976, 275, 50001))])
def test_state_dict_keys_and_shapes_match_the_reference(name, shapes):
    """Keys/shapes recorded from the live reference (SURVEY.md 8b; oracle shape tables are pinned by the golden tests)."""
    import importlib
    import config
    Model = getattr(importlib.import_module(f"model.{name}"), name)
    m = Model(getattr(config, name + "Config"))
    sd = m.state_dict()
    want = shapes()
    assert set(sd.keys()) == set(want.keys())
    for k, shp in want.items():
        assert tuple(sd[k].shape) == tuple(shp), k
        assert sd[k].dtype == torch.float32
    for meth in ("forward", "get_news_vector", "get_user_vector", "get_prediction"):
        assert callable(getattr(m, meth))
    assert "NewsEncoder" in repr(m)  # print(model) works (train.py:109)


def test_naml_shares_one_word_table_and_one_category_table():
    import config
    from model.NAML import NAML
    m = NAML(config.NAMLConfig)
    te, ee = m.news_encoder.text_encoders, m.news_encoder.element_encoders
    assert te["title"].word_embedding.weight.data_ptr() == te["abstract"].word_embedding.weight.data_ptr()
    assert ee["category"].embedding.weight.data_ptr() == ee["subcategory"].embedding.weight.data_ptr()


def test_checkpoint_round_trip_between_state_dicts(tmp_path):
    import config
    from model.NRMS import NRMS
    cfg = type("C", (config.NRMSConfig,), dict(num_words=50))
    a, b = NRMS(cfg), NRMS(cfg)
    torch.save({"model_state_dict": a.state_dict(), "step": 3}, tmp_path / "ckpt-3.pth")
    b.load_state_dict(torch.load(tmp_path / "ckpt-3.pth")["model_state_dict"])
    for k, v in a.state_dict().items():
        assert torch.equal(v, b.state_dict()[k]), k


def test_slot_packer_orders_browsed_block_then_candidates():
    from newsrec_b200.pack import SlotPacker
    B, C, H, T = 3, 2, 4, 5
    cand = [{"title": torch.full((B, T), 100 + j) + torch.arange(B).view(B, 1)} for j in range(C)]
    clicked = [{"title": torch.full((B, T), 200 + j) + torch.arange(B).view(B, 1)} for j in range(H)]
    ids, b = SlotPacker().pack(clicked, cand, "title", torch.device("cpu"))
    assert b == B and ids.shape == (B * H + B * C, T)
    assert ids[:B * H].view(B, H, T)[1, 2, 0] == 200 + 2 + 1       # impression 1, history slot 2
    assert ids[B * H:].view(B, C, T)[2, 1, 0] == 100 + 1 + 2       # impression 2, candidate 1
    # twice through the double-buffered staging keeps results independent
    ids2, _ = SlotPacker().pack(clicked, cand, "title", torch.device("cpu"))
    assert torch.equal(ids, ids2)


def test_operand_cache_rebuilds_only_when_the_parameter_changes():
    from newsrec_b200.ops import OperandCache
    cache, calls = OperandCache(), []
    p = torch.nn.Parameter(torch.zeros(4))
    build = lambda t: calls.append(1) or t.clone()
    cache.get("w", (p,), build)
    cache.get("w", (p,), build)
    assert len(calls) == 1
    with torch.no_grad():
        p.add_(1.0)            # what optimizer.step() does: bumps the version counter
    out = cache.get("w", (p,), build)
    assert len(calls) == 2 and float(out[0]) == 1.0


def test_operand_cache_invalidate_keeps_parameter_independent_workspaces():
    """bench.py drops the parameter-derived operands every step (what an optimizer update does through the version counters);
    workspaces keyed by no parameter (persistent gradient accumulators) must survive."""
    from newsrec_b200.ops import OperandCache
    cache, calls = OperandCache(), []
    p = torch.nn.Parameter(torch.zeros(4))
    cache.get("w", (p,), lambda t: calls.append("w") or t.clone())
    ws = cache.get("ws", (), lambda: calls.append("ws") or torch.zeros(2))
    cache.invalidate_operands()
    cache.get("w", (p,), lambda t: calls.append("w") or t.clone())
    assert cache.get("ws", (), lambda: calls.append("ws") or torch.zeros(2)) is ws
    assert calls == ["w", "ws", "w"]


def test_qkv_sections_pad_to_a_16_byte_phase():
    """Q | K | V sections start at multiples of 8 columns (abi.cu qkv_section): the packed projection operands carry zero rows
    at the section padding, the gradient slices skip it."""
    from newsrec_b200.ops import qkv_pitches, stack_qkv
    assert qkv_pitches(300) == (304, 912) and qkv_pitches(40) == (40, 128) and qkv_pitches(100) == (104, 320)
    Wq, Wk, Wv = (torch.full((300, 300), float(i + 1)) for i in range(3))
    W = stack_qkv(Wq, Wk, Wv)
    assert W.shape == (912, 300)
    for i in range(3):
        assert bool((W[i * 304:i * 304 + 300] == i + 1).all()) and bool((W[i * 304 + 300:(i + 1) * 304] == 0).all())
    b = stack_qkv(torch.ones(300), 2 * torch.ones(300), 3 * torch.ones(300))
    assert b.shape == (912,) and float(b[303]) == 0.0 and float(b[304]) == 2.0 and float(b[911]) == 0.0
    assert stack_qkv(torch.ones(40, 40), torch.ones(40, 40), torch.ones(40, 40)).shape == (120, 40)  # d % 8 == 0: no padding


def test_precision_knob_defaults_and_validation():
    """config.precision: "accurate" by default for NRMS and LSTUR (the blueprint's 1e-3 tolerance), "fast" on request;
    the removed fused_news_encoder knob and anything else are rejected."""
    import config as cfgmod
    from newsrec_b200 import NewsrecError
    from newsrec_b200.ops import precision_mode
    assert precision_mode(cfgmod.NRMSConfig) == os.environ.get("NEWSREC_PRECISION", "accurate")
    assert getattr(cfgmod.LSTURConfig, "precision") == os.environ.get("NEWSREC_PRECISION", "accurate")
    assert precision_mode(type("C", (), {"precision": "fast"})) == "fast"
    with pytest.raises(NewsrecError):
        precision_mode(type("C", (), {"precision": "fast", "fused_news_encoder": True}))
    assert precision_mode(type("C", (), {})) == "fast"  # a config without the knob (NAML / TANR): plain bf16 storage
    with pytest.raises(NewsrecError):
        precision_mode(type("C", (), {"precision": "exact"}))


def test_hot_path_raises_without_cuda_instead_of_falling_back():
    if torch.cuda.is_available():
        pytest.skip("CUDA present")
    import config
    from model.NRMS import NRMS
    from newsrec_b200 import NewsrecError
    cfg = type("C", (config.NRMSConfig,), dict(num_words=30))
    m = NRMS(cfg)
    with pytest.raises(NewsrecError):
        m.get_news_vector({"title": torch.zeros(2, 20, dtype=torch.long)})
    with pytest.raises(NewsrecError):
        m.get_prediction(torch.zeros(3, 300), torch.zeros(300))


def test_product_package_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "news-recommendation_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                text = open(os.path.join(dirpath, f), errors="ignore").read()
                assert "newsrec_oracle" not in text and "oracle/" not in text.replace("the oracle", ""), os.path.join(dirpath, f)


def test_shard_range_partitions_exactly():
    from newsrec_b200.ddp import shard_range
    for n, w in ((4096, 8), (10, 3), (7, 8)):
        spans = [shard_range(n, r, w) for r in range(w)]
        assert spans[0][0] == 0 and spans[-1][1] == n
        assert all(a[1] == b[0] for a, b in zip(spans, spans[1:]))
        assert max(hi - lo for lo, hi in spans) - min(hi - lo for lo, hi in spans) <= 1


def _ddp_worker(rank, world, port, q):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    sys.path.insert(0, os.path.join(ROOT, "news-recommendation_b200", "src"))
    from newsrec_b200 import ddp
    r, w, _ = ddp.init_from_env("gloo")
    torch.manual_seed(0)
    a, b = torch.nn.Parameter(torch.randn(5, 3)), torch.nn.Parameter(torch.randn(7))
    fg = ddp.FlatGradients([a, b, a], w)          # duplicate (tied) parameter appears once
    assert a.grad.data_ptr() == fg.flat.data_ptr()
    # rank-local loss = mean over the local shard of a global batch of 8 samples
    x = torch.arange(8.0).view(8, 1)
    lo, hi = ddp.shard_range(8, r, w)
    fg.zero()
    loss = ((a.sum() + b.sum()) * x[lo:hi]).mean()
    loss.backward()
    fg.all_reduce_mean()
    q.put((r, a.grad.tolist(), b.grad.tolist()))  # plain lists: a tensor would travel as a shared-memory handle that dies with this process
    torch.distributed.destroy_process_group()


def test_flat_gradient_views_start_on_16_byte_boundaries():
    """The kernels accumulate into .grad with 16-byte vector reductions: every view of the flat buffer must be aligned,
    whatever the parameter sizes are (odd sizes get padding behind them)."""
    import torch
    from newsrec_b200 import ddp
    from newsrec_b200.ops import grad_sink
    ps = [torch.nn.Parameter(torch.randn(*shape)) for shape in ((5, 3), (7,), (2, 2), (1,), (9, 300))]
    fg = ddp.FlatGradients(ps, 1)
    for p in ps:
        assert p.grad.data_ptr() % 16 == 0 and p.grad.is_contiguous() and p.grad.shape == p.shape
        assert grad_sink(p) is p.grad
    # views do not overlap: writing one leaves the others zero
    fg.zero()
    ps[1].grad.fill_(1.0)
    assert float(fg.flat.sum()) == 7.0 and all(float(p.grad.abs().sum()) == 0.0 for i, p in enumerate(ps) if i != 1)
    # a parameter without usable gradient storage is not a sink
    q = torch.nn.Parameter(torch.randn(4))
    assert grad_sink(q) is None
    q.grad = torch.zeros(8)[::2]
    assert grad_sink(q) is None
    # direct accumulation is an opt-in of the storage's owner: a .grad that merely exists (a plain earlier backward,
    # optimizer.zero_grad(set_to_none=False)) is NOT written in place -- AccumulateGrad and its hooks keep working
    q.grad = torch.zeros(4)
    assert grad_sink(q) is None


def test_flat_gradient_all_reduce_equals_single_process_mean_gloo():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + (os.getpid() % 400)
    procs = [ctx.Process(target=_ddp_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    want = torch.arange(8.0).mean()   # d/dtheta of mean_i (theta_sum * x_i) over the GLOBAL batch
    for _, ga, gb in got:
        assert torch.allclose(torch.tensor(ga), torch.full((5, 3), float(want))) and torch.allclose(torch.tensor(gb), torch.full((7,), float(want)))


def test_bench_synthetic_batches_are_mind_shaped():
    sys.path.insert(0, ROOT)
    import bench
    _, cand, clicked = bench.synth_slots("NRMS", 6, 3)
    assert len(cand) == 5 and len(clicked) == 50 and cand[0]["title"].shape == (6, 20) and cand[0]["title"].dtype == torch.int64
    hist = torch.stack([x["title"] for x in clicked], 1)             # (B, 50, 20)
    empty = (hist.sum(-1) == 0)
    assert bool((empty[:, :-1] | ~empty[:, 1:]).all()) or True       # left padding: empty slots precede real ones
    first_real = (~empty).float().argmax(1)
    for b in range(6):
        assert bool(empty[b, :first_real[b]].all()) and not bool(empty[b, first_real[b]:].any())
    t = cand[0]["title"]
    nz = (t != 0)
    assert bool((nz[:, :-1] | ~nz[:, 1:]).all())                     # titles right padded with 0
    assert int(t.max()) < bench.V_WORDS and bench.usable_cores() >= 1
    f, b = bench.kernel_work("news.fwd/gemm_store[563200,900,300]")
    assert f == 2.0 * 563200 * 900 * 300 and b > 0
    # the other BASELINE configurations: every attribute the model reads, LSTUR's record fields, left-padded history
    extra, cand, clicked = bench.synth_slots("LSTUR", 4, 5)
    assert set(cand[0]) == {"category", "subcategory", "title"} and extra[0].shape == (4,) and int(extra[1].min()) >= 1
    _, cand, clicked = bench.synth_slots("NAML", 4, 5)
    assert cand[0]["abstract"].shape == (4, 50) and clicked[0]["category"].shape == (4,)
    hl = (torch.stack([x["title"] for x in clicked], 1).sum(-1) != 0).sum(1)
    assert bool((torch.stack([x["category"] for x in clicked], 1) != 0).sum(1).eq(hl).all())  # empty news are empty in every field
    assert abs(bench.flop_fwd_per_impression("NRMS", 300) / 1e6 - 789.5) < 0.5
