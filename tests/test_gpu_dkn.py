"""DKN on the H100: the drop-in against the golden case and the oracle, the KCNN encoder kernel pair at several shapes against
the fp64 oracle under its storage contract, the history-attention kernels through the C ABI against fp64, get_prediction and
device evaluation.

Element bounds of nr_dkn_user_*: every output is a chain of at most three fp32 products summed over at most n = max(F, H) terms,
and the softmax takes the dot products s_j = beta . h_j, whose absolute error e ~ sqrt(F) u max|beta| max|h| is a relative error
e of the weights.  So |got - ref| <= 16 sqrt(F H) u (1 + max|s|) max|ref| (as test_gpu_hifiark, u = 2^-24).
"""
import math
import os

import numpy as np
import pytest
import torch

import dkn_oracle as DO
import newsrec_oracle as O
from golden_util import V, load_case

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
U = 2.0 ** -24


def lib():
    from newsrec_b200 import load_library
    return load_library()


def _p(t):
    import ctypes as C
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def relerr(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm())


def centred(x):
    return x - x.mean(dim=1, keepdim=True)


def make_cfg(VE, **kw):
    import config
    return type("Cfg", (config.DKNConfig,), dict(dict(num_words=V, num_entities=VE, num_clicked_news_a_user=6), **kw))


GOLDEN = {"dkn": (2, 3, 4), "dkn_w4133": (4, 1, 3, 3)}  # golden case -> config.window_sizes it was minted at


def build(g, windows=DO.WINDOWS):
    from model.DKN import DKN
    VE = int(g["num_entities"])
    torch.manual_seed(0)
    model = DKN(make_cfg(VE, window_sizes=list(windows))).to(DEV)
    model.load_state_dict(DO.dkn_state_dict(V, VE, int(g["seed"]), windows=windows))
    return model


def params(g, requires_grad=True, dtype=torch.float32, windows=DO.WINDOWS):
    return {k: v.to(dtype).clone().requires_grad_(requires_grad)
            for k, v in DO.dkn_state_dict(V, int(g["num_entities"]), int(g["seed"]), windows=windows).items()}


def ids(g):
    return [torch.from_numpy(g[k]) for k in ("cand_title", "cand_entities", "clicked_title", "clicked_entities")]


def slots(t, e):
    return [{"title": t[:, j].contiguous(), "title_entities": e[:, j].contiguous()} for j in range(t.shape[1])]


def _check_golden_case(case):
    g, win = load_case(case), GOLDEN[case]
    model = build(g, win).train()  # DKN has no dropout: train and eval mode compute the same
    ct, ce, ht, he = ids(g)
    p_b, p_x = params(g, windows=win), params(g, windows=win)
    lb = DO.dkn_forward(ct, ce, ht, he, p_b, O.BF16, win)[0]
    O.click_loss(lb).backward()
    lx = DO.dkn_forward(ct, ce, ht, he, p_x, O.EXACT, win)[0]
    O.click_loss(lx).backward()
    with torch.no_grad():
        lw = DO.dkn_forward(ct, ce, ht, he, params(g, False, windows=win), O.WEIGHTS_BF16, win)[0]
    logits = model(slots(ct, ce), slots(ht, he))
    loss = torch.nn.functional.cross_entropy(logits, torch.zeros(logits.shape[0], dtype=torch.long, device=DEV))
    loss.backward()
    torch.cuda.synchronize()
    res = {"contract": relerr(logits, lb), "contract_centred": relerr(centred(logits), centred(lb)),
           "weights_bf16": relerr(logits, lw), "weights_bf16_centred": relerr(centred(logits), centred(lw)),
           "golden": relerr(logits, torch.from_numpy(g["logits"]))}
    print(case, "golden", res)
    assert res["contract"] < 1e-3 and res["contract_centred"] < 1e-3, res
    assert res["weights_bf16"] < 1e-3 and res["golden"] < 3e-3, res
    Fp = len(win) * 50
    worst = 0.0
    for k, prm in model.named_parameters():
        exact = p_x[k].grad
        if k in ("attention.dnn.0.bias", "attention.dnn.1.bias"):  # analytically zero: exact zeros, not rounding noise
            assert prm.grad is not None and bool((prm.grad == 0).all()), k
            continue
        if k == "click_predictor.dnn.2.bias":
            # adds one constant to every logit of an impression, and the cross-entropy's logit gradients sum to 0 over the
            # candidates: the exact gradient is 0, and every evaluation of it (fp32 oracle, contract, kernels) rounding noise
            assert float(prm.grad.abs().max()) <= 1e-6 and float(exact.abs().max()) <= 1e-6, (k, prm.grad, exact)
            continue
        if k == "attention.dnn.0.weight":
            assert bool((prm.grad[:, :Fp] == 0).all()), k
            got, exact, contract = prm.grad[:, Fp:], exact[:, Fp:], p_b[k].grad[:, Fp:]
        else:
            got, contract = prm.grad, p_b[k].grad
        e_k = relerr(got, exact)
        e_c = float((contract - exact).norm() / exact.norm())
        worst = max(worst, e_k / max(e_c, 2e-3))
        assert e_k <= 1.5 * max(e_c, 2e-3), (k, e_k, e_c)
    print("worst gradient error over the contract's", worst)
    assert bool((model.kcnn.word_embedding.weight.grad[0] == 0).all())
    assert bool((model.kcnn.entity_embedding.weight.grad[0] == 0).all())


def test_golden_case():
    _check_golden_case("dkn")


def test_golden_case_at_windows_4133():
    """unsorted windows, a repeated size, window 1 and window 4"""
    _check_golden_case("dkn_w4133")


# ---- the KCNN encoder kernel pair against the fp64 oracle under its contract ---------------------------------------------------
def kcnn_case(n, T, VE, entities, seed):
    title = O.synth_titles(n, T, V, seed, min_len=min(T, 5))
    if entities == "zero":
        ents = torch.zeros_like(title)
    elif entities == "last":  # the last row of both tables
        title[:, 0] = V - 1
        ents = DO.synth_entities(title, VE, seed + 3)
        ents[:, 0] = VE - 1
    else:
        ents = DO.synth_entities(title, VE, seed + 3)
    return title, ents


def _kcnn_param(n, T, entities, windows=DO.WINDOWS, tag=None):
    # the cases at the default windows keep the ids they had before the window sets were added
    return pytest.param(n, T, entities, windows, id=f"{n}-{T}-{entities}" + (f"-{tag}" if tag else ""))


@pytest.mark.parametrize("n,T,entities,windows", [
    _kcnn_param(96, 20, "mixed"),      # MIND title length
    _kcnn_param(70, 4, "mixed"),       # T = the widest window: one position for it
    _kcnn_param(9, 64, "mixed"),       # T = 64: whole pooling tiles per title
    _kcnn_param(37, 23, "mixed"),      # segments of 22 / 21 / 20 rows crossing 64-row tiles
    _kcnn_param(40, 20, "zero"),       # no entity anywhere: the entity scatter has no live tile
    _kcnn_param(40, 20, "last"),       # id = V - 1 in both tables
    _kcnn_param(96, 20, "mixed", (1,), "w1"),                 # one window of one tap
    _kcnn_param(96, 20, "mixed", (4, 2), "w42"),              # unsorted: the news vector keeps the list's order
    _kcnn_param(96, 20, "mixed", (3, 3), "w33"),              # a repeated size: one conv, two blocks, two gradient parts
    _kcnn_param(96, 20, "mixed", (1, 2, 3, 4), "w1234"),      # four windows
    _kcnn_param(96, 20, "mixed", (4, 1, 3, 3), "w4133")])     # the second golden case's windows
def test_kcnn_encoder_against_fp64_contract(n, T, entities, windows):
    from model.DKN.KCNN import KCNN
    VE = 30
    cfg = make_cfg(VE, num_words_title=T, window_sizes=list(windows))
    torch.manual_seed(0)
    enc = KCNN(cfg, None, None, None).to(DEV)
    sd = {k[len("kcnn."):]: v for k, v in DO.dkn_state_dict(V, VE, 7, windows=windows).items() if k.startswith("kcnn.")}
    enc.load_state_dict(sd)
    title, ents = kcnn_case(n, T, VE, entities, 1000 + T)
    dout = O.det_uniform((n, 50 * len(windows)), 77, -1, 1, torch.float64)
    p_c = {"kcnn." + k: v.double().clone().requires_grad_(True) for k, v in sd.items()}
    p_x = {"kcnn." + k: v.double().clone().requires_grad_(True) for k, v in sd.items()}
    want = DO.kcnn(title, ents, p_c, O.BF16, windows)
    (want * dout).sum().backward()
    exact = DO.kcnn(title, ents, p_x, O.EXACT, windows)
    (exact * dout).sum().backward()
    got = enc.encode_ids(title.to(DEV), ents.to(DEV))
    (got * dout.float().to(DEV)).sum().backward()
    torch.cuda.synchronize()
    assert int(enc._flag.get(DEV).item()) == 0
    got, want = got.detach().double().cpu(), want.detach()
    # forward: the kernels store the same bf16 sites as the contract, so what is left is accumulation order and the tanh
    # approximation, plus an occasional stored value rounding to the neighbouring bf16 (one ulp, 2^-8 relative)
    assert relerr(got, want) < 2e-3, relerr(got, want)
    assert float((got - want).abs().max()) <= 2.0 ** -7 * float(want.abs().max()), float((got - want).abs().max())
    for k, prm in enc.named_parameters():
        key = "kcnn." + k
        if float(p_x[key].grad.norm()) == 0.0:  # no live entity id: nothing may be scattered
            assert bool((prm.grad == 0).all()), key
            continue
        e_k = relerr(prm.grad, p_x[key].grad)
        e_c = float((p_c[key].grad - p_x[key].grad).norm() / p_x[key].grad.norm())
        assert e_k <= 1.5 * max(e_c, 2e-3), (key, e_k, e_c)
    assert bool((enc.word_embedding.weight.grad[0] == 0).all()) and bool((enc.entity_embedding.weight.grad[0] == 0).all())


def test_kcnn_bad_ids_set_the_flag():
    from model.DKN.KCNN import KCNN
    enc = KCNN(make_cfg(30), None, None, None).to(DEV)
    for bad_title, bad_ent in ((V, 0), (1, 30), (-1, 0)):
        title = torch.ones((4, 20), dtype=torch.int64, device=DEV)
        ents = torch.zeros_like(title)
        title[2, 3], ents[1, 5] = bad_title, bad_ent
        enc._flag = type(enc._flag)()
        enc.encode_ids(title, ents)
        torch.cuda.synchronize()
        assert int(enc._flag.get(DEV).item()) == 1, (bad_title, bad_ent)


def test_kcnn_refuses_shapes_outside_its_bounds():
    from newsrec_b200 import NewsrecError
    from model.DKN.KCNN import KCNN
    enc = KCNN(make_cfg(30, num_words_title=3), None, None, None).to(DEV)
    title = torch.ones((4, 3), dtype=torch.int64, device=DEV)  # T = 3 < the widest window
    with pytest.raises(NewsrecError):
        enc.encode_ids(title, torch.zeros_like(title))
    with pytest.raises(NewsrecError):
        KCNN(make_cfg(30, use_context=True), None, None, None)


def test_kcnn_refuses_a_window_of_5_before_any_launch():
    """The reference accepts any window size; the kernels take 1 to 4 taps (include/newsrec_b200.h), so the drop-in refuses
    a wider window when it is built, not at the first batch."""
    from newsrec_b200 import NewsrecError
    from model.DKN import DKN
    from model.DKN.KCNN import KCNN
    l0 = int(lib().nr_launch_count())
    for wins in ([5], [2, 3, 5], [0, 2]):
        with pytest.raises(NewsrecError, match="window"):
            KCNN(make_cfg(30, window_sizes=wins), None, None, None)
        with pytest.raises(NewsrecError, match="window"):
            DKN(make_cfg(30, window_sizes=wins))
    assert int(lib().nr_launch_count()) == l0


# ---- nr_dkn_user_* through the C ABI --------------------------------------------------------------------------------------------
class Guarded:
    """A device buffer of n floats (NaN, or 0.0 for += outputs) followed by a guard band no call may touch."""

    def __init__(self, shape, fill=float("nan")):
        n = int(np.prod(shape))
        self.buf = torch.full((n + 256,), fill, dtype=torch.float32, device=DEV)
        self.t = self.buf[:n].view(shape)

    def guard_ok(self):
        band = self.buf[self.t.numel():]
        return bool(torch.isnan(band).all()) if bool(torch.isnan(self.buf[-1])) else bool((band == self.buf[-1]).all())


@pytest.mark.parametrize("B,H,F,Hd", [(5, 50, 156, 16), (3, 1, 150, 16), (2, 64, 512, 32), (4, 7, 1, 1)])
def test_dkn_user_kernels_against_fp64(B, H, F, Hd):
    from newsrec_b200 import check
    x = O.det_uniform((B, H, F), 11, -1, 1, torch.float64) * 2
    W1 = O.det_uniform((Hd, 2 * F), 12, -0.5, 0.5, torch.float64)
    w2 = O.det_uniform((Hd,), 13, -1, 1, torch.float64)
    du = O.det_uniform((B, F), 14, -1, 1, torch.float64)
    xr, W1r, w2r = (t.clone().requires_grad_(True) for t in (x, W1, w2))
    beta = torch.matmul(w2r, W1r[:, F:])
    s = torch.matmul(xr, beta)
    u = torch.bmm(torch.softmax(s, 1).unsqueeze(1), xr).squeeze(1)
    (u * du).sum().backward()
    xd, W1d, w2d, dud = (t.float().to(DEV).contiguous() for t in (x, W1, w2, du))
    user, dhist = Guarded((B, F)), Guarded((B, H, F))
    dW1, dw2 = Guarded((Hd, 2 * F), 0.0), Guarded((Hd,), 0.0)
    check(lib().nr_dkn_user_fwd(_p(xd), B, H, F, _p(W1d), Hd, _p(w2d), _p(user.t), None), "nr_dkn_user_fwd")
    ws_bytes = int(lib().nr_dkn_user_bwd_workspace(B, F))
    ws = torch.full((ws_bytes // 4,), float("nan"), device=DEV)
    check(lib().nr_dkn_user_bwd(_p(xd), B, H, F, _p(W1d), Hd, _p(w2d), _p(dud), _p(dhist.t), _p(dW1.t), _p(dw2.t), _p(ws), ws_bytes,
                                None), "nr_dkn_user_bwd")
    torch.cuda.synchronize()
    assert all(b.guard_ok() for b in (user, dhist, dW1, dw2))
    smax = float(s.abs().max())
    for name, g, w in (("user", user.t, u), ("dhist", dhist.t, xr.grad), ("dW1", dW1.t, W1r.grad), ("dw2", dw2.t, w2r.grad)):
        g, w = g.double().cpu(), w.detach()
        assert torch.isfinite(g).all(), name
        tol = 16 * math.sqrt(F * H) * U * (1 + smax) * max(w.abs().max().item(), 1e-30) * (B if name in ("dW1", "dw2") else 1)
        assert float((g - w).abs().max()) <= tol, (name, float((g - w).abs().max()), tol)
    assert bool((dW1.t[:, :F] == 0).all())  # the candidate half: exact zeros
    # the weight gradients are summed in a fixed order: a second run adds bit-identical values
    before = (dW1.t.clone(), dw2.t.clone())
    check(lib().nr_dkn_user_bwd(_p(xd), B, H, F, _p(W1d), Hd, _p(w2d), _p(dud), _p(dhist.t), _p(dW1.t), _p(dw2.t), _p(ws), ws_bytes,
                                None), "nr_dkn_user_bwd")
    torch.cuda.synchronize()
    assert torch.equal(dW1.t, 2 * before[0]) and torch.equal(dw2.t, 2 * before[1])


def test_dkn_user_refuses_shapes_outside_its_bounds():
    x = torch.zeros((1, 65, 513), device=DEV)
    W = torch.zeros((33, 1026), device=DEV)
    ws = torch.zeros(1 << 20, dtype=torch.uint8, device=DEV)
    l0 = int(lib().nr_launch_count())
    for H, F, Hd in ((0, 8, 16), (65, 8, 16), (6, 0, 16), (6, 513, 16), (6, 8, 0), (6, 8, 33)):
        assert lib().nr_dkn_user_fwd(_p(x), 1, H, F, _p(W), Hd, _p(W), _p(x), None) == -2, (H, F, Hd)
        assert b"supported bounds" in lib().nr_last_error()
        assert lib().nr_dkn_user_bwd(_p(x), 1, H, F, _p(W), Hd, _p(W), _p(x), _p(x), _p(W), _p(W), _p(ws), ws.numel(), None) == -2
    assert int(lib().nr_launch_count()) == l0


# ---- get_prediction and evaluation -------------------------------------------------------------------------------------------
def test_get_prediction_matches_the_oracle():
    g = load_case("dkn")
    model = build(g).eval()
    p = params(g, False, torch.float64)
    cv, hv = torch.from_numpy(g["cand_vec"]), torch.from_numpy(g["clicked_vec"])
    with torch.no_grad():
        for b in range(cv.shape[0]):
            want = DO.get_prediction(cv[b].double(), hv[b].double(), p)
            got = model.get_prediction(cv[b].to(DEV), hv[b].to(DEV))
            assert got.shape == (cv.shape[1],)
            np.testing.assert_allclose(got.cpu().double().numpy(), want.numpy(), rtol=1e-5, atol=1e-6)
            np.testing.assert_allclose(want.numpy(), g["pred"][b], rtol=1e-5, atol=1e-6)
        assert model.get_user_vector(hv.to(DEV)) is not None


def test_device_evaluation_matches_the_oracle_loop(tmp_path):
    """evaluate() on synthetic MIND files: every impression's scores against the fp64 oracle's get_prediction on the same
    news vectors and (left-padded) histories, and the metrics against their per-impression restatement."""
    import ranking_metrics as R
    import test_gpu_evaluate as TE
    from newsrec_b200 import evaluate as E
    from model.DKN import DKN
    d = str(tmp_path)
    TE._write_validation_dir(d)
    cfg = make_cfg(30, num_words=TE.V, num_clicked_news_a_user=TE.H, batch_size=2)
    torch.manual_seed(0)
    model = DKN(cfg).to(DEV).eval()
    with torch.no_grad():  # entity rows non-trivial although the synthetic titles carry no entity
        model.kcnn.entity_embedding.weight[0].uniform_(-1, 1)
    pd_ = {k: v.detach().double().cpu() for k, v in model.state_dict().items()}
    u2i = os.path.join(d, "user2int.tsv")
    with torch.no_grad():
        index, matrix = E.news_matrix(model, d)
        tables = E.build_tables(d, index, TE.H, 10 ** 9, u2i)
        flag = E.new_flag(DEV)
        users = E.user_vectors(model, tables, matrix, flag)
        assert users.dim() == 3
        scores = E.impression_scores(tables, matrix, users, flag, model).cpu().double()
        assert int(flag.item()) == 0
    m = matrix.double().cpu()
    offs, tasks = tables.seg_offsets, []
    for s in range(len(tables.seg_user)):
        hist = m[torch.from_numpy(tables.history[tables.seg_user[s]])]
        cand = m[torch.from_numpy(tables.cand[offs[s]:offs[s + 1]])]
        y = DO.get_prediction(cand, hist, pd_)
        np.testing.assert_allclose(scores[offs[s]:offs[s + 1]].numpy(), y.numpy(), rtol=1e-5, atol=1e-6)
        tasks.append((tables.labels[offs[s]:offs[s + 1]].astype(int).tolist(), y.tolist()))
    ref = np.nanmean(np.array([R.single_impression(y, t) for t, y in tasks]), axis=0)
    got = E.evaluate(model, d, 4, user2int_path=u2i)
    assert np.abs(np.array(got) - ref).max() <= 1e-6, (got, ref)
