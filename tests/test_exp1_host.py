"""Exp1 without a GPU: the oracle against golden vectors of the live reference (tests/golden/exp1.npz), the storage contracts
against the blueprint's tolerance, and the drop-in's configuration and state_dict surface."""
import importlib
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import newsrec_oracle as O
from exp1_util import exp1_params, golden_grad_key, load, oracle_logits, relerr
from golden_util import grad_summary, unique_params

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG_SRC = os.path.join(ROOT, "news-recommendation_b200", "src")


def test_oracle_matches_reference_fp32():
    g = load()
    p = exp1_params(g)
    logits = oracle_logits(g, p)
    np.testing.assert_allclose(logits.detach().numpy(), g["logits"], rtol=2e-5, atol=2e-5)
    loss = O.click_loss(logits)
    assert abs(loss.item() - float(g["loss"])) < 2e-5 * max(1.0, abs(float(g["loss"])))
    loss.backward()
    checked = set()
    gscale = max(float(g[k][0]) for k in g if k.startswith("gsum:"))
    for k, prm in unique_params(p).items():
        key = golden_grad_key(k, g)
        assert key is not None, f"no golden gradient for {k}"
        s, samp = grad_summary(prm.grad, key)
        ref_s, ref_samp = g["gsum:" + key], g["gsamp:" + key]
        if ref_s[0] < 1e-4 * gscale:  # analytically zero (W_K.bias: a per-query constant cancels in the softmax): rounding noise
            assert s[0] < 1e-4 * gscale, (k, s, ref_s)
            continue
        scale = max(ref_s[0], 1e-3)
        assert abs(s[0] - ref_s[0]) <= 1e-4 * scale, (k, s, ref_s)
        assert abs(s[1] - ref_s[1]) <= 1e-4 * scale, (k, s, ref_s)
        np.testing.assert_allclose(samp, ref_samp, rtol=1e-3, atol=2e-5 * scale)
        checked.add(k)
    assert "user_encoder.position_embedding" in checked
    assert "news_encoder.element_encoders.category.embedding.weight" in checked  # the shared table, once
    assert float(p["user_encoder.position_embedding"].grad.norm()) > 0
    assert float(p["user_encoder.position_embedding"].detach().abs().max()) <= 0.1  # the reference's init scale


def test_storage_contracts_against_the_blueprint_tolerance():
    """Norm-wise distance of the logits from the fp32 oracle on bf16-rounded weights: the shipped ("accurate") contract is
    inside 1e-3, the plain-bf16 ("fast") one is not better."""
    g = load()
    p = exp1_params(g, requires_grad=False)
    with torch.no_grad():
        want = oracle_logits(g, p, O.WEIGHTS_BF16)
        acc = relerr(oracle_logits(g, p, "accurate"), want)
        fast = relerr(oracle_logits(g, p, "fast"), want)
    assert acc < 1e-3, acc
    assert fast > acc, (fast, acc)


def test_positional_gradient_is_the_input_gradient_summed_over_users():
    """dpos = sum over the batch of d(hv + pos): what the kernels reduce (fp64, exact contract)."""
    g = load()
    p = exp1_params(g, dtype=torch.float64)
    hv = torch.from_numpy(g["clicked_vec"]).double().requires_grad_(True)
    import exp1_oracle as E
    E.exp1_user_encoder(hv, p).sum().backward()
    torch.testing.assert_close(p["user_encoder.position_embedding"].grad, hv.grad.sum(0), rtol=1e-12, atol=1e-12)


def _drop_in_config(**over):
    if PKG_SRC not in sys.path:
        sys.path.insert(0, PKG_SRC)
    import config as cfgmod
    base = dict(num_words=120, num_categories=15, num_clicked_news_a_user=6)
    base.update(over)
    return type("Cfg", (cfgmod.Exp1Config,), base)


def test_drop_in_state_dict_has_the_golden_keys_and_shapes():
    import exp1_oracle as E
    g = load()
    cfg = _drop_in_config()
    Exp1 = importlib.import_module("model.Exp1").Exp1
    sd = Exp1(cfg).state_dict()
    want = E.exp1_shapes(120, 15, 6)
    assert set(sd) == set(want)
    assert all(tuple(sd[k].shape) == tuple(v) for k, v in want.items())
    m = Exp1(cfg)
    ne = m.news_encoder
    assert ne.element_encoders["category"].embedding is ne.element_encoders["subcategory"].embedding
    m.load_state_dict(E.exp1_state_dict(120, 15, 6, int(g["seed"])))
    assert cfg.precision in ("accurate", "fast") and cfg.ensemble_factor == 1 and cfg.num_attention_heads == 15


def test_model_name_exp1_imports_config_and_abstract_is_refused():
    env = dict(os.environ, MODEL_NAME="Exp1", PYTHONPATH=PKG_SRC)
    r = subprocess.run([sys.executable, "-c", "import config; c = config.Exp1Config; "
                        "print(c.dataset_attributes['news'], c.num_attention_heads, c.ensemble_factor, c.precision)"],
                       env=env, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert "['category', 'subcategory', 'title'] 15 1 accurate" in r.stdout
    from newsrec_b200 import NewsrecError
    Exp1 = importlib.import_module("model.Exp1").Exp1
    cfg = _drop_in_config(dataset_attributes={"news": ["category", "subcategory", "title", "abstract"], "record": []})
    with pytest.raises(NewsrecError, match="abstract"):
        Exp1(cfg)


def test_history_length_must_match_the_position_embedding():
    from newsrec_b200 import NewsrecError
    Exp1 = importlib.import_module("model.Exp1").Exp1
    m = Exp1(_drop_in_config())
    with pytest.raises(NewsrecError, match="num_clicked_news_a_user"):
        m.get_user_vector(torch.zeros(2, 5, 300))
