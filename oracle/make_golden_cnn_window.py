"""Golden vectors of the CNN text encoders at conv windows other than 3, from the LIVE reference modules (build container only),
in make_golden.py's format:

    PYTHONHASHSEED=0 python oracle/make_golden_cnn_window.py [case ...]      (default: every case in CASES)

Each case (tests/golden/<case>.npz) is built as make_golden.py / make_golden_hifiark.py build a family's case -- the same
shapes, input synthesis and deterministic state_dict -- at another window_size and with its own seed; the fixture records the
window (window_size):
    naml_w4       NAML, both text encoders at window 4 (title L = 19, abstract L = 49)
    tanr_w1       TANR at window 1 (the topic head included)
    lstur_ini_w2  LSTUR ini at window 2
    hifiark_w2    Hi-Fi Ark at window 2 (+ the regulariser and the 1-D get_prediction scores, as hifiark.npz)
The reference asserts an odd window in LSTUR, TANR and Hi-Fi Ark (NAML does not): at an even window the model is built at
window 3 and every window-3 text conv replaced by the Conv2d the reference's own expression makes at the case's window
(reference_at_window).  Forward + CrossEntropy(label 0) + backward in .eval() mode on CPU fp32.
"""
from __future__ import annotations

import importlib
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import hifiark_oracle as HO  # noqa: E402
import make_golden as MG  # noqa: E402
import newsrec_oracle as O  # noqa: E402

CASES = {"naml_w4": ("NAML", 21, 4), "tanr_w1": ("TANR", 22, 1), "lstur_ini_w2": ("LSTUR", 23, 2), "hifiark_w2": ("HiFiArk", 24, 2)}
META = f"torch={torch.__version__} threads={torch.get_num_threads()} ref=8323a4f"


def reference_at_window(name, cfg, window):
    """The reference model `name` at `window`; see the module docstring for even windows."""
    Model = getattr(importlib.import_module("model." + name), name)
    if window % 2 == 1 or name == "NAML":
        return Model(cfg)
    model = Model(type(cfg.__name__, (cfg,), {"window_size": 3}))
    for mod in list(model.modules()):
        for child, conv in list(mod.named_children()):
            if isinstance(conv, torch.nn.Conv2d) and conv.kernel_size[0] == 3 and conv.in_channels == 1:
                setattr(mod, child, torch.nn.Conv2d(1, conv.out_channels, (window, conv.kernel_size[1]),
                                                    padding=(int((window - 1) / 2), 0)))
    return model


def categories(seed, clicked_t, sub=True):
    """make_golden.py's category / subcategory ids of the candidates and the browsed news."""
    B, C, H, NCAT = MG.B, MG.C, MG.H, MG.NCAT
    out = dict(cand_category=O.det_randint((B, C), seed * 100 + 60, 1, NCAT))
    if sub:
        out["cand_subcategory"] = O.det_randint((B, C), seed * 100 + 61, 1, NCAT)
    out["clicked_category"] = O.det_randint((B, H), seed * 100 + 62, 1, NCAT) * (clicked_t[..., 0] > 0)
    if sub:
        out["clicked_subcategory"] = O.det_randint((B, H), seed * 100 + 63, 1, NCAT) * (clicked_t[..., 0] > 0)
    return out


def news_slots(prefix, fields):
    """Reference slot lists: one dict of (B,) / (B, T) tensors per slot."""
    names = [k for k in ("title", "abstract", "category", "subcategory") if f"{prefix}_{k}" in fields]
    n = fields[prefix + "_title"].shape[1]
    return [{k: fields[f"{prefix}_{k}"][:, j].contiguous() for k in names} for j in range(n)]


def add_grads(rec, model):
    seen = set()
    for k, prm in model.named_parameters():
        if prm.grad is None or id(prm) in seen:
            continue
        seen.add(id(prm))
        rec["gsum:" + k], rec["gsamp:" + k] = MG.grad_summary(prm.grad, k)


def save(case, rec, loss, logits):
    path = os.path.join(MG.OUT, f"{case}.npz")
    np.savez_compressed(path, **rec)
    print(f"{case}: loss={loss.item():.6f} logits[0]={logits[0].tolist()} -> {case}.npz ({os.path.getsize(path) / 1024:.0f} KB)")


def run_family(case):
    """NAML / TANR / LSTUR: make_golden.run_case's recording at the case's window."""
    name, seed, window = CASES[case]
    B, C, H, T, TA, V, NCAT, NUSERS = MG.B, MG.C, MG.H, MG.T, MG.TA, MG.V, MG.NCAT, MG.NUSERS
    cand_t, clicked_t, hist_len = O.synth_batch(B, C, H, T, V, seed * 100)
    fields = dict(cand_title=cand_t, clicked_title=clicked_t)
    args = ()
    if name == "NAML":
        cfg = MG.make_config("NAML", window_size=window,
                             dataset_attributes={"news": ["category", "subcategory", "title", "abstract"], "record": []})
        shapes = O.naml_shapes(V, NCAT, window=window)
        ca, ha, _ = O.synth_batch(B, C, H, TA, V, seed * 100 + 50)
        extra = dict(cand_abstract=ca * (cand_t[..., :1] > 0), clicked_abstract=ha * (clicked_t[..., :1] > 0), **categories(seed, clicked_t))
    elif name == "TANR":
        cfg = MG.make_config("TANR", window_size=window, dataset_attributes={"news": ["category", "title"], "record": []})
        shapes = O.tanr_shapes(V, NCAT, window=window)
        extra = categories(seed, clicked_t, sub=False)
    else:
        cfg = MG.make_config("LSTUR", window_size=window, long_short_term_method="ini",
                             dataset_attributes={"news": ["category", "subcategory", "title"], "record": ["user", "clicked_news_length"]})
        shapes = O.lstur_shapes(V, NCAT, NUSERS, window=window, method="ini")
        lengths = hist_len.clone()
        lengths[0] = 0  # the reference's 0 -> 1 clamp (LSTUR/user_encoder.py:27), as make_golden.py
        extra = dict(categories(seed, clicked_t), user=O.det_randint((B,), seed * 100 + 70, 1, NUSERS), clicked_news_length=lengths)
        args = (extra["user"], lengths.clone())
    fields.update(extra)
    sd = O.tie_shared(O.det_state_dict(shapes, seed))
    model = reference_at_window(name, cfg, window)
    missing = set(model.state_dict().keys()) ^ set(sd.keys())
    assert not missing, f"state_dict key mismatch for {case}: {sorted(missing)}"
    model.load_state_dict(sd)
    model.eval()
    news_vecs, user_vecs = [], []
    model.news_encoder.register_forward_hook(lambda m, i, o: news_vecs.append(o.detach()))
    model.user_encoder.register_forward_hook(lambda m, i, o: user_vecs.append(o.detach()))
    out = model(*args, news_slots("cand", fields), news_slots("clicked", fields))
    logits, topic_loss = out if isinstance(out, tuple) else (out, None)
    loss = torch.nn.functional.cross_entropy(logits, torch.zeros(B, dtype=torch.long))
    (loss + (0.1 * topic_loss if topic_loss is not None else 0.0)).backward()
    rec = dict(cand_title=cand_t.numpy(), clicked_title=clicked_t.numpy(), hist_len=hist_len.numpy(),
               logits=logits.detach().numpy(), loss=np.array(loss.item()), cand_vec=torch.stack(news_vecs[:C], dim=1).numpy(),
               clicked_vec=torch.stack(news_vecs[C:C + H], dim=1).numpy(), user_vec=user_vecs[0].numpy(), seed=np.array(seed),
               meta=np.array(META))
    if topic_loss is not None:
        rec["topic_loss"] = np.array(topic_loss.item())
    rec["window_size"] = np.array(window)
    for k, v in extra.items():
        rec[k] = v.numpy()
    add_grads(rec, model)
    save(case, rec, loss, logits)


def run_hifiark(case):
    """make_golden_hifiark.run's recording at the case's window."""
    _, seed, window = CASES[case]
    B, C, H, T, V = MG.B, MG.C, MG.H, MG.T, MG.V
    cand_t, clicked_t, hist_len = O.synth_batch(B, C, H, T, V, seed * 100)
    cfg = MG.make_config("HiFiArk", num_pooling_heads=5, regularizer_loss_weight=0.1, window_size=window)
    model = reference_at_window("HiFiArk", cfg, window)
    sd = O.det_state_dict(HO.hifiark_shapes(V, window=window), seed, {"omap.W": 0.1})  # hifiark_state_dict at the window
    missing = set(model.state_dict().keys()) ^ set(sd.keys())
    assert not missing, f"state_dict key mismatch for {case}: {sorted(missing)}"
    model.load_state_dict(sd)
    model.eval()
    fields = dict(cand_title=cand_t, clicked_title=clicked_t)
    news_vecs, archives = [], []
    model.news_encoder.register_forward_hook(lambda m, i, o: news_vecs.append(o.detach()))
    model.omap.register_forward_hook(lambda m, i, o: archives.append(o[0].detach()))
    logits, reg_eval = model(news_slots("cand", fields), news_slots("clicked", fields))
    assert reg_eval is None
    loss = torch.nn.functional.cross_entropy(logits, torch.zeros(B, dtype=torch.long))
    loss.backward()
    cand_vec, clicked_vec, archive = torch.stack(news_vecs[:C], dim=1), torch.stack(news_vecs[C:C + H], dim=1), archives[0]
    with torch.no_grad():
        pred1d = np.array([[model.get_prediction(cand_vec[b, j], archive[b]).item() for j in range(C)] for b in range(B)])
    rec = dict(cand_title=cand_t.numpy(), clicked_title=clicked_t.numpy(), hist_len=hist_len.numpy(),
               logits=logits.detach().numpy(), loss=np.array(loss.item()), cand_vec=cand_vec.numpy(), clicked_vec=clicked_vec.numpy(),
               archive=archive.numpy(), pred1d=pred1d, seed=np.array(seed), meta=np.array(META))
    add_grads(rec, model)
    model.zero_grad()  # the regulariser: model.omap in train mode (OMAP.py:36-44), its gradient alone
    model.omap.train()
    _, reg = model.omap(cand_vec.detach())
    reg.backward()
    rec["reg"] = np.array(reg.item())
    rec["reg_gsum"], rec["reg_gsamp"] = MG.grad_summary(model.omap.W.grad, "reg:omap.W")
    rec["window_size"] = np.array(window)
    save(case, rec, loss, logits)


if __name__ == "__main__":
    assert os.path.isdir(MG.REF_SRC), "the reference is only mounted in the build container"
    sys.path.insert(0, MG.REF_SRC)
    for case in sys.argv[1:] or CASES:
        torch.manual_seed(0)
        (run_hifiark if CASES[case][0] == "HiFiArk" else run_family)(case)
