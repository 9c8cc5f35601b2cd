"""Exp1 on the H100: the drop-in against the golden vectors of the live reference and the oracle's storage contracts (eval and
train mode, accurate and fast), the kernels it adds (positional addend, its deterministic gradient, the one-pass hi/lo split),
device evaluation, ensembles, and an ensemble under data parallel with one FlatGradients per model.

Tolerances are those of tests/test_gpu_models.py: logits within 1e-3 of the oracle under the kernels' storage contract and of
the fp32 oracle on bf16-rounded weights, within 1.25 x the contract's own error (+1e-4) of the reference's fp32 logits, every
gradient's error against the exact gradient within 1.5 x the contract's own (floor 2e-3)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

import exp1_oracle as E
import newsrec_oracle as O
from exp1_util import H, exp1_fields, exp1_params, load, oracle_logits, relerr, slot_lists
from golden_util import NCAT, V, unique_params

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build(V=V, ncat=NCAT, H=H, precision="accurate", dropout=0.2, seed=None):
    import config as cfgmod
    from model.Exp1 import Exp1
    cfg = type("Cfg", (cfgmod.Exp1Config,), dict(num_words=V, num_categories=ncat, num_clicked_news_a_user=H,
                                                 dropout_probability=dropout, precision=precision))
    model = Exp1(cfg)
    if seed is not None:
        model.load_state_dict(E.exp1_state_dict(V, ncat, H, seed))
    return model.to(DEV), cfg


def _grad_ratios(model, p_x, p_b, res):
    """kernel error / contract error of every gradient against the exact one (floor 2e-3); analytically ~0 ones skipped."""
    grads = dict(model.named_parameters(remove_duplicate=False))
    gscale = max(float(v.grad.norm()) for v in unique_params(p_x).values())
    worst, worst_key = 0.0, ""
    for k, prm in unique_params(p_x).items():
        gk = grads[k].grad
        if gk is None:
            res["missing_grad:" + k] = True
            continue
        if prm.grad.norm() < 1e-4 * gscale:
            continue
        e_kernel, e_contract = relerr(gk, prm.grad), relerr(unique_params(p_b)[k].grad, prm.grad)
        res["grad:" + k] = [e_kernel, e_contract]
        ratio = e_kernel / max(e_contract, 2e-3)
        if ratio > worst:
            worst, worst_key = ratio, k
    res["worst_grad_ratio_kernel_over_contract"], res["worst_grad_key"] = worst, worst_key
    res["emb_row0_grad_zero"] = bool((grads["news_encoder.text_encoders.title.word_embedding.weight"].grad[0] == 0).all())
    return res


def check_golden(precision, train=False, p_drop=0.2):
    from newsrec_b200 import ops
    g = load()
    model, _ = build(precision=precision, dropout=p_drop, seed=int(g["seed"]))
    drop = None
    if train:
        model.train()
        drop = dict(p=p_drop, seed=ops.peek_seeds(1)[0])  # the title encoder is the batch's only dropout draw
    else:
        model.eval()
    p_b = exp1_params(g)
    logits_b = oracle_logits(g, p_b, precision, drop)
    O.click_loss(logits_b).backward()
    p_x = exp1_params(g)
    logits_x = oracle_logits(g, p_x, O.EXACT, drop)
    O.click_loss(logits_x).backward()
    cand, clicked = slot_lists(g)
    logits = model(cand, clicked)
    torch.nn.functional.cross_entropy(logits, torch.zeros(logits.shape[0], dtype=torch.long, device=DEV)).backward()
    torch.cuda.synchronize()
    with torch.no_grad():
        logits_w = oracle_logits(g, exp1_params(g, requires_grad=False), O.WEIGHTS_BF16, drop)
        logits_eval = oracle_logits(g, exp1_params(g, requires_grad=False), O.EXACT)
    ref = logits_x if train else torch.from_numpy(g["logits"])
    res = {"logits_vs_oracle_contract": relerr(logits, logits_b), "logits_vs_weights_only_oracle": relerr(logits, logits_w),
           "logits_vs_reference_fp32": relerr(logits, ref), "oracle_contract_vs_reference_fp32": relerr(logits_b, ref),
           "masks_matter": relerr(logits_x, logits_eval)}
    return _grad_ratios(model, p_x, p_b, res)


def _assert_golden(r):
    assert r["logits_vs_oracle_contract"] < 1e-3, r
    assert r["logits_vs_reference_fp32"] < 1.25 * r["oracle_contract_vs_reference_fp32"] + 1e-4, r
    assert r["worst_grad_ratio_kernel_over_contract"] < 1.5, r
    assert "grad:user_encoder.position_embedding" in r, r
    assert r["emb_row0_grad_zero"], r
    assert not any(k.startswith("missing_grad:") for k in r), r


def test_golden_case_accurate():
    r = check_golden("accurate")
    _assert_golden(r)
    assert r["logits_vs_weights_only_oracle"] < 1e-3, r  # the blueprint's tolerance


def test_golden_case_fast():
    r = check_golden("fast")
    _assert_golden(r)


@pytest.mark.parametrize("precision", ["accurate", "fast"])
def test_train_mode_matches_masked_oracle(precision):
    r = check_golden(precision, train=True)
    assert r["masks_matter"] > 0.05, r
    _assert_golden(r)


# ------------------------------------------------------------------------------------------------------------------------
# kernel level
# ------------------------------------------------------------------------------------------------------------------------
def _dense_forward_planes(x, pos, accurate):
    """nr_mhsa_encoder_fwd on the dense variant with random operands: returns (X_bf16, X_kcat_bf16 or None)."""
    from newsrec_b200 import MhsaEncoderFwdArgs, check, load_library
    from newsrec_b200.ops import OperandCache, _p, _stream, cast_pad, mhsa_operands, qkv_pitches, ru8, stack_qkv
    lib = load_library()
    n_seq, T, d = x.shape
    q, heads = 200, 15
    ldx = ru8(d + 1)
    sec, ld3 = qkv_pitches(d)
    gen = torch.Generator().manual_seed(1)
    W = [torch.randn(d, d, generator=gen) * 0.05 for _ in range(3)]
    b = [torch.randn(d, generator=gen) * 0.05 for _ in range(3)]
    Wa, ba, qv = torch.randn(q, d, generator=gen) * 0.05, torch.randn(q, generator=gen) * 0.05, torch.randn(q, generator=gen) * 0.1
    prm = [t.to(DEV) for t in (W[0], b[0], W[1], b[1], W[2], b[2], Wa, ba, qv)]
    ops = mhsa_operands(OperandCache(), "t", *prm)
    n_tok = n_seq * T
    a = MhsaEncoderFwdArgs()
    a.n_seq, a.T, a.d, a.heads, a.q, a.ldx, a.ld3 = n_seq, T, d, heads, q, ldx, ld3
    a.dense = _p(x)
    a.dense_s_seq, a.dense_s_tok, a.dense_s_col = x.stride()
    a.wqkv_bf16, a.bqkv, a.wa_bf16, a.ba, a.qv = _p(ops["wqkv"]), _p(ops["bqkv"]), _p(ops["wa"]), _p(ops["ba"]), _p(ops["qv"])
    X = torch.full((n_tok, ldx), 7.0, dtype=torch.bfloat16, device=DEV)  # sentinel: every element must be written
    Cx = torch.empty((n_tok, ldx), dtype=torch.bfloat16, device=DEV)
    w = torch.empty((n_tok,), dtype=torch.float32, device=DEV)
    out = torch.empty((n_seq, d), dtype=torch.float32, device=DEV)
    keep = [X, Cx, w, out]
    kcat = None
    if accurate:
        wk = cast_pad(torch.cat((torch.nn.functional.pad(stack_qkv(*prm[0:6:2]), (0, ldx - d)),) * 2, dim=1), 2 * ldx)
        kcat = torch.full((n_tok, 2 * ldx), 7.0, dtype=torch.bfloat16, device=DEV)
        qf = torch.empty((n_tok, 3 * sec), dtype=torch.float32, device=DEV)
        clo = torch.empty((n_tok, ldx), dtype=torch.bfloat16, device=DEV)
        keep += [wk, qf, clo]
        a.wqkv_kcat_bf16, a.X_kcat_bf16, a.QKV_f32, a.C_lo_bf16 = _p(wk), _p(kcat), _p(qf), _p(clo)
        a.QKV_bf16 = None
    else:
        QKV = torch.empty((n_tok, ld3), dtype=torch.bfloat16, device=DEV)
        keep.append(QKV)
        a.QKV_bf16 = _p(QKV)
    a.X_bf16, a.C_bf16, a.w, a.out = _p(X), _p(Cx), _p(w), _p(out)
    a.dense_pos = _p(pos) if pos is not None else None
    check(lib.nr_mhsa_encoder_fwd(C.byref(a), _stream()), "nr_mhsa_encoder_fwd")
    torch.cuda.synchronize()
    return X, kcat


def _want_rows(xs, ldx):
    """bf16 rows + ones column at d, zeros after (what the conversion kernels write for fp32 rows xs (n, d))."""
    n, d = xs.shape
    want = torch.zeros((n, ldx), dtype=torch.bfloat16, device=xs.device)
    want[:, :d] = xs.to(torch.bfloat16)
    want[:, d] = 1.0
    return want


def _bits(t):
    return t.view(torch.int16)


@pytest.mark.parametrize("accurate", [True, False])
def test_dense_pos_null_and_set_give_the_defined_bits(accurate):
    n_seq, T, d = 37, 50, 300
    base = torch.randn(T, n_seq, d + 7, device=DEV) * 2.0
    x = base.transpose(0, 1)[:, :, 3:3 + d]  # non-contiguous: (n_seq, T, d) with strides (d+7, n_seq*(d+7), 1)
    x[0, 0, :3] = torch.tensor([-0.0, 3.0e38, -7.5], device=DEV)
    assert not x.is_contiguous()
    ldx = (d + 8) // 8 * 8
    pos = (torch.rand(T, d, device=DEV) * 0.2 - 0.1).contiguous()
    for p in (None, pos):
        X, kcat = _dense_forward_planes(x, p, accurate)
        xs = (x if p is None else x + p).reshape(n_seq * T, d)  # fp32 sum, then the one rounding
        want = _want_rows(xs, ldx)
        assert torch.equal(_bits(X), _bits(want)), p is None
        if accurate:
            assert torch.equal(_bits(kcat[:, :ldx]), _bits(X))  # hi plane == X_bf16, bitwise
            lo = torch.zeros_like(X)
            lo[:, :d] = (xs - xs.to(torch.bfloat16).float()).to(torch.bfloat16)
            assert torch.equal(_bits(kcat[:, ldx:]), _bits(lo))


def test_positional_gradient_is_deterministic_and_sums_the_input_gradient():
    """B=512, H=50, d=300: dpos is reduced on the device in a fixed order, not with atomics."""
    B, T, d = 512, 50, 300
    model, _ = build(V=50, H=T, precision="accurate", seed=3)
    ue = model.user_encoder
    hv = (torch.randn(B, T, d, device=DEV) * 0.3).requires_grad_(True)
    dout = torch.randn(B, d, device=DEV)
    grads = []
    for _ in range(2):
        ue.position_embedding.grad = None
        hv.grad = None
        ue(hv).backward(dout)
        torch.cuda.synchronize()
        grads.append((ue.position_embedding.grad.clone(), hv.grad.clone()))
    assert torch.equal(grads[0][0], grads[1][0])  # bit-identical across runs
    want = grads[0][1].double().sum(0)
    err = float((grads[0][0].double() - want).abs().max() / want.abs().max())
    assert err < 1e-5, err  # fp32 summation noise
    assert torch.isfinite(grads[0][0]).all() and float(want.abs().max()) > 0


def test_hilo_split_kernel():
    from newsrec_b200 import check, load_library
    from newsrec_b200.ops import _p, _stream
    lib = load_library()
    n, D, ld = 4099, 300, 304
    x = torch.randn(n, D + 5, device=DEV)[:, 2:2 + D] * torch.logspace(-3, 3, D, device=DEV)
    hi = torch.full((n, ld), 7.0, dtype=torch.bfloat16, device=DEV)
    lo = torch.full((n, ld), 7.0, dtype=torch.bfloat16, device=DEV)
    check(lib.nr_rows_to_bf16_hilo(_p(x), n, D, x.stride(0), x.stride(1), _p(hi), _p(lo), ld, _stream()), "nr_rows_to_bf16_hilo")
    torch.cuda.synchronize()
    assert torch.equal(_bits(hi), _bits(_want_rows(x, ld)))
    assert (lo[:, D:] == 0).all()
    rel = ((hi[:, :D].float() + lo[:, :D].float()) - x).abs() / x.abs().clamp_min(1e-30)
    assert float(rel.max()) <= 2.0 ** -16, float(rel.max())


# ------------------------------------------------------------------------------------------------------------------------
# device evaluation, ensembles
# ------------------------------------------------------------------------------------------------------------------------
def test_device_evaluator_matches_the_reference_loop(tmp_path):
    import ranking_metrics as R
    import test_gpu_evaluate as TE
    from newsrec_b200 import evaluate as EV
    d = str(tmp_path)
    TE._write_validation_dir(d)
    torch.manual_seed(0)
    model, cfg = build(V=TE.V, ncat=TE.NCAT, H=TE.H, seed=5)
    cfg.batch_size = 2
    attrs = list(cfg.dataset_attributes["news"])
    model.eval()
    u2i = os.path.join(d, "user2int.tsv")
    max_count = 10 ** 9
    with torch.no_grad():
        news2vector, user2vector, tasks = TE._reference_loop(model, d, attrs, max_count)
        index, matrix = EV.news_matrix(model, d)
        tables = EV.build_tables(d, index, TE.H, max_count, u2i)
        flag = EV.new_flag(DEV)
        users = EV.user_vectors(model, tables, matrix, flag)
        scores = EV.impression_scores(tables, matrix, users, flag)
        torch.cuda.synchronize()
        assert int(flag.item()) == 0
    ids = [k for k in news2vector if k != "PADDED_NEWS"]
    assert torch.equal(matrix[[index[k] for k in ids]].cpu(), torch.stack([news2vector[k] for k in ids]).cpu())
    hist_strings = list(user2vector)
    assert len(hist_strings) == len(tables.user)
    ref_u = torch.stack([user2vector[s] for s in hist_strings])
    assert TE._rel(users[torch.arange(len(hist_strings))], ref_u) <= 1e-6
    offs = tables.seg_offsets
    assert len(offs) - 1 == len(tasks)
    worst = 0.0
    for s, (y_true, y_pred) in enumerate(tasks):
        got = scores[offs[s]:offs[s + 1]].cpu().double()
        worst = max(worst, TE._rel(got, torch.tensor(y_pred, dtype=torch.float64)))
        assert list(tables.labels[offs[s]:offs[s + 1]]) == y_true
        p = np.sort(np.asarray(y_pred))
        assert (np.diff(p) > 1e-5 * np.maximum(np.abs(p[1:]), np.abs(p[:-1]))).all(), (s, y_pred)
    assert worst <= 1e-6, worst
    for k in (max_count, 17):
        sub = tasks[:k - 1]
        ref = np.nanmean(np.array([R.single_impression(y_pred, y_true) for y_true, y_pred in sub]), axis=0)
        got = EV.evaluate(model, d, 4, k, user2int_path=u2i)
        assert np.abs(np.array(got) - ref).max() <= 1e-6, (got, ref)


def test_ensemble_matches_the_oracle_ensemble():
    """train.py:192-200: NLLLoss(log(mean softmax)) over two independent instances (different weights)."""
    g = load()
    seeds = (int(g["seed"]), int(g["seed"]) + 1)
    models = [build(seed=s)[0].eval() for s in seeds]
    cand, clicked = slot_lists(g)
    logits = [m(cand, clicked) for m in models]
    E.ensemble_loss(logits).backward()
    torch.cuda.synchronize()
    cf, hf = exp1_fields(g)
    p_b = [E.exp1_state_dict(V, NCAT, H, s) for s in seeds]
    p_x = [E.exp1_state_dict(V, NCAT, H, s) for s in seeds]
    leaves = lambda sd: {k: v for k, v in sd.items()}
    ob, ox = [], []
    for pb, px in zip(p_b, p_x):
        for sd in (pb, px):
            seen = {}
            for k, v in list(sd.items()):
                sd[k] = seen.setdefault(id(v), v.clone().requires_grad_(True))
        ob.append(E.exp1_forward(cf, hf, pb, 15, "accurate"))
        ox.append(E.exp1_forward(cf, hf, px, 15, O.EXACT))
    E.ensemble_loss(ob).backward()
    E.ensemble_loss(ox).backward()
    for i, m in enumerate(models):
        assert relerr(logits[i], ob[i]) < 1e-3
        assert relerr(logits[i], ox[i]) < 1.25 * relerr(ob[i], ox[i]) + 1e-4
        r = _grad_ratios(m, leaves(p_x[i]), leaves(p_b[i]), {})
        assert r["worst_grad_ratio_kernel_over_contract"] < 1.5, (i, r)
        assert not any(k.startswith("missing_grad:") for k in r), r
    # independent operand caches and gradients
    t0, t1 = (m.news_encoder.text_encoders["title"] for m in models)
    assert t0._cache is not t1._cache and models[0].user_encoder._cache is not models[1].user_encoder._cache
    k0 = {n: v[1] for n, v in t0._cache._store.items()}
    k1 = {n: v[1] for n, v in t1._cache._store.items()}
    assert k0["news"]["wqkv"].data_ptr() != k1["news"]["wqkv"].data_ptr()
    assert not torch.equal(k0["news"]["wqkv"], k1["news"]["wqkv"])
    pe = [m.user_encoder.position_embedding.grad for m in models]
    assert pe[0].data_ptr() != pe[1].data_ptr() and not torch.equal(pe[0], pe[1])


# ------------------------------------------------------------------------------------------------------------------------
# two GPUs: an ensemble under data parallel, one FlatGradients per model
# ------------------------------------------------------------------------------------------------------------------------
def _ddp_worker(rank, world, port, out_dir):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    for p in (os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle"), os.path.join(ROOT, "news-recommendation_b200", "src")):
        sys.path.insert(0, p)
    global DEV
    from newsrec_b200 import ddp
    torch.cuda.set_device(rank)
    DEV = torch.device("cuda", rank)
    r, w, _ = ddp.init_from_env("nccl")
    Bn, Cn, Hn, T, Vn = 16, 5, 50, 20, 3000
    models = [build(V=Vn, ncat=NCAT, H=Hn, seed=s)[0].eval() for s in (3, 4)]
    refs = [build(V=Vn, ncat=NCAT, H=Hn, seed=s)[0].eval() for s in (3, 4)]  # plain autograd gradients, no communication
    flats = [ddp.FlatGradients(m.parameters(), w) for m in models]
    pad4 = lambda n: (n + 3) // 4 * 4
    results = []
    for step in range(3):
        cand_t, clicked_t, _ = O.synth_batch(Bn, Cn, Hn, T, Vn, 100 * step + r)
        cats = [O.det_randint(shape, 1000 * step + 10 * r + j, 1, NCAT) for j, shape in enumerate(((Bn, Cn),) * 2 + ((Bn, Hn),) * 2)]
        mk = lambda t, c, s: [{"title": t[:, j].contiguous(), "category": c[:, j].contiguous(), "subcategory": s[:, j].contiguous()}
                              for j in range(t.shape[1])]
        cand, clicked = mk(cand_t, cats[0], cats[1]), mk(clicked_t, cats[2], cats[3])
        for m in refs:
            m.zero_grad(set_to_none=True)
        E.ensemble_loss([m(cand, clicked) for m in refs]).backward()
        for f in flats:
            f.zero()
        E.ensemble_loss([m(cand, clicked) for m in models]).backward()
        for f in flats:
            f.all_reduce_mean()  # no synchronisation before: model 0's early slice must wait for ITS scatter GEMM
        torch.cuda.synchronize()
        per_model = []
        for m, ref, f in zip(models, refs, flats):
            name_of = {id(prm): k for k, prm in m.named_parameters()}
            rp = dict(ref.named_parameters())
            local = torch.zeros_like(f.flat)
            off = 0
            for prm in f.params:
                n = prm.numel()
                local[off:off + n] = rp[name_of[id(prm)]].grad.reshape(-1)
                off += pad4(n)
            per_model.append((local.cpu(), f.flat.clone().cpu()))
        results.append(per_model)
    torch.save(results, os.path.join(out_dir, f"rank{r}.pt"))
    torch.distributed.barrier()
    torch.distributed.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_ensemble_all_reduce_with_one_flat_buffer_per_model(tmp_path):
    import torch.multiprocessing as mp
    mp.spawn(_ddp_worker, args=(2, 29573, str(tmp_path)), nprocs=2, join=True)
    r0, r1 = torch.load(tmp_path / "rank0.pt"), torch.load(tmp_path / "rank1.pt")
    for step, (m0, m1) in enumerate(zip(r0, r1)):
        for i, ((l0, a0), (l1, a1)) in enumerate(zip(m0, m1)):
            assert torch.equal(a0, a1), (step, i)
            want = (l0.double() + l1.double()) / 2
            scale = float(want.abs().max())
            err = float((a0.double() - want).abs().max()) / scale
            assert err < 2e-5, (step, i, err)
            assert float((l0 - l1).abs().max()) > 1e-3 * scale
