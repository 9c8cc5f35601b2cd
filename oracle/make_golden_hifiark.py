"""Golden vectors of Hi-Fi Ark from the LIVE reference modules (build container only), in make_golden.py's format:

    PYTHONHASHSEED=0 python oracle/make_golden_hifiark.py

One case (tests/golden/hifiark.npz): B=3, 1+K=3, H=6, P=5 on the shapes of make_golden.py, a deterministic state_dict
(hifiark_oracle.hifiark_state_dict), forward + CrossEntropy(label 0) + backward in .eval() mode on CPU fp32 (the reference's
eval-mode forward returns None for the regulariser).  The regulariser and its gradient come from model.omap in train mode on
its own; the 1-D get_prediction scores of every (user, candidate) pair are recorded as well.
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

SEED = 18


def run():
    sys.path.insert(0, MG.REF_SRC)
    B, C, H, T, V = MG.B, MG.C, MG.H, MG.T, MG.V
    cand_t, clicked_t, hist_len = O.synth_batch(B, C, H, T, V, SEED * 100)
    cfg = MG.make_config("HiFiArk", num_pooling_heads=5, regularizer_loss_weight=0.1)
    model = importlib.import_module("model.HiFiArk").HiFiArk(cfg)
    sd = HO.hifiark_state_dict(V, SEED)
    missing = set(model.state_dict().keys()) ^ set(sd.keys())
    assert not missing, f"state_dict key mismatch for hifiark: {sorted(missing)}"
    model.load_state_dict(sd)
    model.eval()
    cand = [{"title": x} for x in MG.slots(cand_t)]
    clicked = [{"title": x} for x in MG.slots(clicked_t)]
    news_vecs, archives = [], []
    model.news_encoder.register_forward_hook(lambda m, i, o: news_vecs.append(o.detach()))
    model.omap.register_forward_hook(lambda m, i, o: archives.append(o[0].detach()))
    logits, reg_eval = model(cand, clicked)
    assert reg_eval is None
    loss = torch.nn.functional.cross_entropy(logits, torch.zeros(B, dtype=torch.long))
    loss.backward()
    cand_vec, clicked_vec, archive = torch.stack(news_vecs[:C], dim=1), torch.stack(news_vecs[C:C + H], dim=1), archives[0]
    with torch.no_grad():
        pred1d = np.array([[model.get_prediction(cand_vec[b, j], archive[b]).item() for j in range(C)] for b in range(B)])
    rec = dict(cand_title=cand_t.numpy(), clicked_title=clicked_t.numpy(), hist_len=hist_len.numpy(),
               logits=logits.detach().numpy(), loss=np.array(loss.item()), cand_vec=cand_vec.numpy(), clicked_vec=clicked_vec.numpy(),
               archive=archive.numpy(), pred1d=pred1d, seed=np.array(SEED),
               meta=np.array(f"torch={torch.__version__} threads={torch.get_num_threads()} ref=8323a4f"))
    seen = set()
    for k, prm in model.named_parameters():
        if prm.grad is None or id(prm) in seen:
            continue
        seen.add(id(prm))
        s, samp = MG.grad_summary(prm.grad, k)
        rec["gsum:" + k] = s
        rec["gsamp:" + k] = samp
    # the regulariser: model.omap in train mode (OMAP.py:36-44), its gradient alone
    model.zero_grad()
    model.omap.train()
    _, reg = model.omap(cand_vec.detach())
    reg.backward()
    rec["reg"] = np.array(reg.item())
    rec["reg_gsum"], rec["reg_gsamp"] = MG.grad_summary(model.omap.W.grad, "reg:omap.W")
    path = os.path.join(MG.OUT, "hifiark.npz")
    np.savez_compressed(path, **rec)
    print(f"hifiark: loss={loss.item():.6f} reg={reg.item():.6f} logits[0]={logits[0].tolist()} -> hifiark.npz "
          f"({os.path.getsize(path) / 1024:.0f} KB)")


if __name__ == "__main__":
    assert os.path.isdir(MG.REF_SRC), "the reference is only mounted in the build container"
    torch.manual_seed(0)
    run()
