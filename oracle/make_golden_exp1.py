"""Golden vectors of Exp1 from the LIVE reference modules (build container only), in make_golden.py's format:

    PYTHONHASHSEED=0 python oracle/make_golden_exp1.py

One case (tests/golden/exp1.npz): B=3, 1+K=3, H=6 on the shapes of make_golden.py, title + category + subcategory inputs
(as LSTUR's case), a deterministic state_dict (exp1_oracle.exp1_state_dict), forward + CrossEntropy(label 0) + backward in
.eval() mode on CPU fp32.
"""
from __future__ import annotations

import importlib
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import exp1_oracle as E  # noqa: E402
import make_golden as MG  # noqa: E402
import newsrec_oracle as O  # noqa: E402

SEED = 17


def run():
    sys.path.insert(0, MG.REF_SRC)
    B, C, H, T, V, NCAT = MG.B, MG.C, MG.H, MG.T, MG.V, MG.NCAT
    cand_t, clicked_t, hist_len = O.synth_batch(B, C, H, T, V, SEED * 100)
    cc = O.det_randint((B, C), SEED * 100 + 60, 1, NCAT)
    cs = O.det_randint((B, C), SEED * 100 + 61, 1, NCAT)
    hc = O.det_randint((B, H), SEED * 100 + 62, 1, NCAT) * (clicked_t[..., 0] > 0)
    hs = O.det_randint((B, H), SEED * 100 + 63, 1, NCAT) * (clicked_t[..., 0] > 0)
    cfg = MG.make_config("Exp1", dataset_attributes={"news": ["category", "subcategory", "title"], "record": []},
                         ensemble_factor=1)
    model = importlib.import_module("model.Exp1").Exp1(cfg)
    sd = E.exp1_state_dict(V, NCAT, H, SEED)
    missing = set(model.state_dict().keys()) ^ set(sd.keys())
    assert not missing, f"state_dict key mismatch for exp1: {sorted(missing)}"
    model.load_state_dict(sd)
    model.eval()
    cand = [{"title": a, "category": c_, "subcategory": d_} for a, c_, d_ in zip(MG.slots(cand_t), MG.slots(cc), MG.slots(cs))]
    clicked = [{"title": a, "category": c_, "subcategory": d_} for a, c_, d_ in zip(MG.slots(clicked_t), MG.slots(hc), MG.slots(hs))]
    news_vecs, user_vecs = [], []
    model.news_encoder.register_forward_hook(lambda m, i, o: news_vecs.append(o.detach()))
    model.user_encoder.register_forward_hook(lambda m, i, o: user_vecs.append(o.detach()))
    logits = model(cand, clicked)
    loss = torch.nn.functional.cross_entropy(logits, torch.zeros(B, dtype=torch.long))
    loss.backward()
    rec = dict(cand_title=cand_t.numpy(), clicked_title=clicked_t.numpy(), hist_len=hist_len.numpy(),
               cand_category=cc.numpy(), cand_subcategory=cs.numpy(), clicked_category=hc.numpy(), clicked_subcategory=hs.numpy(),
               logits=logits.detach().numpy(), loss=np.array(loss.item()),
               cand_vec=torch.stack(news_vecs[:C], dim=1).numpy(), clicked_vec=torch.stack(news_vecs[C:C + H], dim=1).numpy(),
               user_vec=user_vecs[0].numpy(), seed=np.array(SEED),
               meta=np.array(f"torch={torch.__version__} threads={torch.get_num_threads()} ref=8323a4f"))
    seen = set()
    for k, prm in model.named_parameters():
        if prm.grad is None or id(prm) in seen:
            continue
        seen.add(id(prm))
        s, samp = MG.grad_summary(prm.grad, k)
        rec["gsum:" + k] = s
        rec["gsamp:" + k] = samp
    path = os.path.join(MG.OUT, "exp1.npz")
    np.savez_compressed(path, **rec)
    print(f"exp1: loss={loss.item():.6f} logits[0]={logits[0].tolist()} -> exp1.npz ({os.path.getsize(path) / 1024:.0f} KB)")


if __name__ == "__main__":
    assert os.path.isdir(MG.REF_SRC), "the reference is only mounted in the build container"
    torch.manual_seed(0)
    run()
