"""Golden vectors of DKN from the LIVE reference modules (build container only), in make_golden.py's format:

    PYTHONHASHSEED=0 python oracle/make_golden_dkn.py [case ...]      (default: every case in CASES)

Each case (tests/golden/<case>.npz): B=3, 1+K=3, H=6 (num_clicked_news_a_user = H: the reference's attention expands the candidate to
that config value) on the shapes of make_golden.py, entity vocabulary VE, title entities mostly 0; a deterministic state_dict
(dkn_oracle.dkn_state_dict), forward + CrossEntropy(label 0) + backward on CPU fp32.  The get_prediction scores of every
user's candidates against its history are recorded as well.  The cases differ in seed and config.window_sizes, which the
fixture records (window_sizes): dkn at the default [2, 3, 4]; dkn_w4133 at [4, 1, 3, 3] -- unsorted, a repeated size (one conv
run twice, its gradient from both) and both ends of the window range.
"""
from __future__ import annotations

import importlib
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import dkn_oracle as DO  # noqa: E402
import make_golden as MG  # noqa: E402
import newsrec_oracle as O  # noqa: E402

VE = 30
CASES = {"dkn": (19, [2, 3, 4]), "dkn_w4133": (20, [4, 1, 3, 3])}  # case -> (seed, window_sizes)


def run(case):
    SEED, windows = CASES[case]
    sys.path.insert(0, MG.REF_SRC)
    B, C, H, T, V = MG.B, MG.C, MG.H, MG.T, MG.V
    cand_t, clicked_t, hist_len = O.synth_batch(B, C, H, T, V, SEED * 100)
    cand_e, clicked_e = DO.synth_entities(cand_t, VE, SEED * 100 + 50), DO.synth_entities(clicked_t, VE, SEED * 100 + 60)
    cfg = MG.make_config("DKN", num_entities=VE, entity_embedding_dim=100, num_filters=50, window_sizes=windows, use_context=False,
                         dataset_attributes={"news": ["title", "title_entities"], "record": []})
    model = importlib.import_module("model.DKN").DKN(cfg)
    sd = DO.dkn_state_dict(V, VE, SEED, windows=windows)
    missing = set(model.state_dict().keys()) ^ set(sd.keys())
    assert not missing, f"state_dict key mismatch for dkn: {sorted(missing)}"
    model.load_state_dict(sd)
    model.eval()
    cand = [{"title": x, "title_entities": e} for x, e in zip(MG.slots(cand_t), MG.slots(cand_e))]
    clicked = [{"title": x, "title_entities": e} for x, e in zip(MG.slots(clicked_t), MG.slots(clicked_e))]
    news_vecs = []
    model.kcnn.register_forward_hook(lambda m, i, o: news_vecs.append(o.detach()))
    logits = model(cand, clicked)
    loss = torch.nn.functional.cross_entropy(logits, torch.zeros(B, dtype=torch.long))
    loss.backward()
    cand_vec, clicked_vec = torch.stack(news_vecs[:C], dim=1), torch.stack(news_vecs[C:C + H], dim=1)
    with torch.no_grad():
        pred = np.stack([model.get_prediction(cand_vec[b], clicked_vec[b]).numpy() for b in range(B)])
    rec = dict(cand_title=cand_t.numpy(), clicked_title=clicked_t.numpy(), cand_entities=cand_e.numpy(),
               clicked_entities=clicked_e.numpy(), hist_len=hist_len.numpy(), num_entities=np.array(VE),
               logits=logits.detach().numpy(), loss=np.array(loss.item()), cand_vec=cand_vec.numpy(), clicked_vec=clicked_vec.numpy(),
               pred=pred, seed=np.array(SEED), window_sizes=np.array(windows), meta=np.array(f"torch={torch.__version__} threads={torch.get_num_threads()} ref=8323a4f"))
    for k, prm in model.named_parameters():
        s, samp = MG.grad_summary(prm.grad, k)
        rec["gsum:" + k] = s
        rec["gsamp:" + k] = samp
    path = os.path.join(MG.OUT, f"{case}.npz")
    np.savez_compressed(path, **rec)
    print(f"{case}: windows={windows} loss={loss.item():.6f} logits[0]={logits[0].tolist()} -> {case}.npz ({os.path.getsize(path) / 1024:.0f} KB)")


if __name__ == "__main__":
    assert os.path.isdir(MG.REF_SRC), "the reference is only mounted in the build container"
    for case in sys.argv[1:] or CASES:
        torch.manual_seed(0)
        run(case)
