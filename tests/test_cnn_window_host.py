"""The CNN text encoders at window_size 1 to 4, without a GPU: the oracle against the window golden cases minted from the live
reference (oracle/make_golden_cnn_window.py), the window check of nr_cnn_encoder_fwd / _bwd (-1 before any
launch, the shape check runs before any pointer is touched) and the refusal of other windows when a model is built."""
import ctypes

import numpy as np
import pytest
import torch

import cnn_window_util as CW
import hifiark_oracle as HO
import newsrec_oracle as O
from golden_util import grad_summary, load_case, unique_params

GOLDEN_CASES = ["naml_w4", "tanr_w1", "lstur_ini_w2"]


@pytest.mark.parametrize("case", sorted(CW.WINDOW_CASES))
def test_fixture_records_its_window(case):
    g = load_case(case)
    w = CW.WINDOW_CASES[case][1]
    assert int(g["window_size"]) == w
    p = CW.case_params(case, g, requires_grad=False)
    assert {v.shape[2] for k, v in p.items() if k.endswith("CNN.weight")} == {w}


def _check_grads(p, g, floor):
    """test_oracle_golden's gradient bounds (tied tensors matched under their sibling name in the reference)."""
    for k, prm in unique_params(p).items():
        key = k if ("gsum:" + k) in g else None
        if key is None:
            sib = {"title": "abstract", "abstract": "title", "category": "subcategory", "subcategory": "category"}
            for a, b in sib.items():
                kk = k.replace(f".{a}.", f".{b}.")
                if ("gsum:" + kk) in g:
                    key = kk
        if key is None:  # Hi-Fi Ark's abstract_CNN: never read, no gradient in the reference either
            assert k.startswith("news_encoder.abstract_CNN") and prm.grad is None, k
            continue
        assert prm.grad is not None, k
        s, samp = grad_summary(prm.grad, key)
        ref_s, ref_samp = g["gsum:" + key], g["gsamp:" + key]
        scale = max(ref_s[0], floor)
        assert abs(s[0] - ref_s[0]) <= 1e-4 * scale, (k, s, ref_s)
        assert abs(s[1] - ref_s[1]) <= 1e-4 * scale, (k, s, ref_s)
        np.testing.assert_allclose(samp, ref_samp, rtol=1e-3, atol=2e-5 * scale)


@pytest.mark.parametrize("case", GOLDEN_CASES)
def test_oracle_matches_reference_fp32_at_window(case):
    """tests/test_oracle_golden.py::test_oracle_matches_reference_fp32 on the window cases."""
    g = load_case(case)
    p = CW.case_params(case, g)
    logits, topic = CW.oracle_forward(case, g, p)
    np.testing.assert_allclose(logits.detach().numpy(), g["logits"], rtol=2e-5, atol=2e-5)
    loss = O.click_loss(logits)
    assert abs(loss.item() - float(g["loss"])) < 2e-5 * max(1.0, abs(float(g["loss"])))
    total = loss
    if topic is not None:
        assert abs(topic.item() - float(g["topic_loss"])) < 2e-5 * max(1.0, abs(float(g["topic_loss"])))
        total = loss + 0.1 * topic
    total.backward()
    _check_grads(p, g, 1e-3)


def test_hifiark_oracle_matches_reference_fp32_at_window_2():
    """tests/test_hifiark_oracle.py::test_oracle_matches_reference_fp32 on hifiark_w2."""
    g = load_case("hifiark_w2")
    p = CW.case_params("hifiark_w2", g)
    ct, ht = torch.from_numpy(g["cand_title"]), torch.from_numpy(g["clicked_title"])
    logits, _, cv, hv, archive = HO.hifiark_forward(ct, ht, p)
    np.testing.assert_allclose(logits.detach().numpy(), g["logits"], rtol=2e-5, atol=2e-5)
    np.testing.assert_allclose(cv.detach().numpy(), g["cand_vec"], rtol=1e-4, atol=1e-5)
    np.testing.assert_allclose(hv.detach().numpy(), g["clicked_vec"], rtol=1e-4, atol=1e-5)
    np.testing.assert_allclose(archive.detach().numpy(), g["archive"], rtol=1e-4, atol=1e-5)
    loss = O.click_loss(logits)
    assert abs(loss.item() - float(g["loss"])) < 2e-5 * max(1.0, abs(float(g["loss"])))
    loss.backward()
    _check_grads(p, g, 5e-2)  # the last DNN bias: analytically zero gradient (test_hifiark_oracle.py)
    assert torch.equal(p["news_encoder.word_embedding.weight"].grad[0], torch.zeros(300))


# ---- the C ABI's window check ----------------------------------------------------------------------------------------------
def _lib():
    import os

    import newsrec_b200
    if not os.path.exists(newsrec_b200.LIB_PATH):
        pytest.skip("library not built (python __graft_entry__.py build)")
    return newsrec_b200.load_library()


def _call(which, T, window, F=400, d=300, q=200):
    import newsrec_b200 as nb
    lib = _lib()
    a = nb.CnnEncoderFwdArgs() if which == "fwd" else nb.CnnEncoderBwdArgs()
    a.n_seq, a.T, a.d, a.F, a.q, a.ldx, a.ldf, a.window = 8, T, d, F, q, (d + 8) // 8 * 8, (F + 8) // 8 * 8, window
    if which == "bwd":
        a.ldq = (q + 15) // 16 * 16
    n0 = lib.nr_launch_count()
    rc = (lib.nr_cnn_encoder_fwd if which == "fwd" else lib.nr_cnn_encoder_bwd)(ctypes.byref(a), None)
    return rc, lib.nr_last_error().decode(), lib.nr_launch_count() - n0


@pytest.mark.parametrize("which", ["fwd", "bwd"])
@pytest.mark.parametrize("window", [5, 6, -1])
def test_window_outside_1_to_4_is_rejected_before_launch(which, window):
    rc, msg, launched = _call(which, 20, window)
    assert rc == -1 and f"window={window}" in msg and launched == 0, (rc, msg, launched)


@pytest.mark.parametrize("which", ["fwd", "bwd"])
@pytest.mark.parametrize("window", [2, 4])
def test_even_window_needs_two_tokens(which, window):
    """T = 1 at an even window leaves no output position (the reference's conv fails there too)."""
    rc, msg, launched = _call(which, 1, window)
    assert rc == -1 and "T=1" in msg and f"window={window}" in msg and launched == 0, (rc, msg, launched)


@pytest.mark.parametrize("which", ["fwd", "bwd"])
@pytest.mark.parametrize("T,window", [(20, 0), (20, 3), (1, 1), (1, 3), (2, 2), (2, 4), (64, 4), (64, 1)])
def test_accepted_windows_pass_the_shape_check(which, T, window):
    """Window 0 means 3; with null operands an accepted shape fails on the pointers instead, still before any launch."""
    rc, msg, launched = _call(which, T, window)
    assert rc == -1 and "null operand" in msg and launched == 0, (rc, msg, launched)


# ---- the drop-in refuses other windows when the model is built ---------------------------------------------------------
@pytest.mark.parametrize("name", ["NAML", "LSTUR", "TANR", "HiFiArk"])
@pytest.mark.parametrize("window", [0, 5])
def test_model_construction_refuses_window(name, window):
    import importlib

    import config as cfgmod
    from newsrec_b200 import NewsrecError
    cfg = type("Cfg", (getattr(cfgmod, name + "Config"),), dict(num_words=50, num_categories=10, num_users=10, window_size=window))
    with pytest.raises(NewsrecError, match=f"window_size={window}"):
        getattr(importlib.import_module("model." + name), name)(cfg)


@pytest.mark.parametrize("name", ["NAML", "LSTUR", "TANR", "HiFiArk"])
@pytest.mark.parametrize("window", [1, 2, 4])
def test_model_construction_takes_windows_1_to_4(name, window):
    import importlib

    import config as cfgmod
    cfg = type("Cfg", (getattr(cfgmod, name + "Config"),), dict(num_words=50, num_categories=10, num_users=10, window_size=window))
    model = getattr(importlib.import_module("model." + name), name)(cfg)
    shapes = {tuple(p.shape) for k, p in model.named_parameters() if k.endswith("CNN.weight")}
    assert shapes == {(cfg.num_filters, 1, window, cfg.word_embedding_dim)}, shapes
