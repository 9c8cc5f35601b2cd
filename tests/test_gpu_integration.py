"""Integration on the H100: every drop-in model driven through the call sequence of the reference's trainer and evaluator.

The reference's drivers cannot travel to the GPU box (and must not be copied), so this test restates ONLY their call
sequence -- each step cites the line it mirrors -- around the drop-in packages:

  train   src/train.py:106 model = Model(config).to(device); :127 Adam(model.parameters()); :183-190 the four forward
          signatures; :202-231 loss = CE(y_pred, 0) (+ 0.1 * topic loss for TANR, :224); loss.backward(); optimizer.step()
  save    src/train.py:264-277 torch.save({'model_state_dict': model.state_dict(), ...}); evaluate.py:287-288 load_state_dict
  eval    src/evaluate.py:193-204 news2vector from get_news_vector over a DataLoader of news dicts (with the "id" list);
          :207-230 get_user_vector over the stacked (NON-contiguous) clicked-news vectors; :245-260 get_prediction per
          impression followed by .tolist()

Batches are built exactly as src/dataset.py:64-85 + torch's default_collate produce them: slot-major lists of dicts of CPU
int64 tensors, history left-padded with all-zero news."""
import io

import pytest
import torch
from torch.utils.data import default_collate

import gpu_checks as G

pytestmark = pytest.mark.gpu

V, NCAT, NUSERS, H, K, T, TA = 300, 12, 40, 50, 4, 20, 50
ATTRS = {"NRMS": ["title"], "NAML": ["category", "subcategory", "title", "abstract"], "LSTUR": ["category", "subcategory", "title"],
         "TANR": ["category", "title"]}


def _news(gen, attrs, empty=False):
    """One parsed news row (src/dataset.py:31-37,70-71); `empty` = the all-zero padding news of a short history (:76-83)."""
    d = {}
    for a in attrs:
        if a in ("title", "abstract"):
            L = T if a == "title" else TA
            ids = torch.zeros(L, dtype=torch.int64)
            if not empty:
                n = int(torch.randint(5, L + 1, (1,), generator=gen))
                ids[:n] = torch.randint(1, V, (n,), generator=gen)
            d[a] = ids
        else:
            d[a] = torch.tensor(0 if empty else int(torch.randint(1, NCAT, (1,), generator=gen)))
    return d


def _sample(gen, attrs, with_record):
    """src/dataset.py:64-85 __getitem__: candidate_news (1+K dicts), clicked_news (H dicts, left-padded), clicked."""
    n_hist = int(torch.randint(0, H + 1, (1,), generator=gen))
    item = {"clicked": [1] + [0] * K, "candidate_news": [_news(gen, attrs) for _ in range(1 + K)],
            "clicked_news": [_news(gen, attrs, empty=True) for _ in range(H - n_hist)] + [_news(gen, attrs) for _ in range(n_hist)]}
    if with_record:
        item["user"] = int(torch.randint(1, NUSERS, (1,), generator=gen))
        item["clicked_news_length"] = n_hist
    return item


def _forward(name, model, mb):
    """src/train.py:183-190."""
    if name == "LSTUR":
        return model(mb["user"], mb["clicked_news_length"], mb["candidate_news"], mb["clicked_news"])
    return model(mb["candidate_news"], mb["clicked_news"])


@pytest.mark.parametrize("name", ["NRMS", "NAML", "LSTUR", "TANR"])
def test_train_checkpoint_evaluate_call_sequence(name):
    case = {"NRMS": "nrms", "NAML": "naml", "LSTUR": "lstur_ini", "TANR": "tanr"}[name]
    gen = torch.Generator().manual_seed(11)
    attrs, dev = ATTRS[name], torch.device("cuda", 0)
    torch.manual_seed(0)
    model, cfg = G.build_model(case, V=V, ncat=NCAT, nusers=NUSERS, H=H)
    optimizer = torch.optim.Adam(model.parameters(), lr=1e-3)                                    # train.py:127
    batches = [default_collate([_sample(gen, attrs, name == "LSTUR") for _ in range(6)]) for _ in range(4)]
    assert isinstance(batches[0]["candidate_news"], list) and batches[0]["candidate_news"][0]["title"].shape == (6, T)
    model.train()
    losses = []
    for step in range(8):                                                                         # train.py:176-231
        mb = batches[step % len(batches)]
        y = _forward(name, model, mb)
        topic = None
        if name == "TANR":
            y, topic = y                                                                           # train.py:190
        loss = torch.nn.functional.cross_entropy(y, torch.zeros(len(y), dtype=torch.long, device=dev))  # :205-206
        if topic is not None:
            loss = loss + cfg.topic_classification_loss_weight * topic                               # :224
        losses.append(loss.item())                                                                 # :225
        optimizer.zero_grad()
        loss.backward()
        optimizer.step()
    assert all(torch.isfinite(torch.tensor(losses))), losses
    assert sum(losses[4:]) < sum(losses[:4]), losses                                               # Adam on 4 repeated batches learns

    buf = io.BytesIO()                                                                            # train.py:264-277
    torch.save({"model_state_dict": model.state_dict(), "optimizer_state_dict": optimizer.state_dict(), "step": 8}, buf)
    buf.seek(0)
    model2, _ = G.build_model(case, V=V, ncat=NCAT, nusers=NUSERS, H=H)
    model2.load_state_dict(torch.load(buf, weights_only=False)["model_state_dict"])              # evaluate.py:287-288
    outs = []
    for mdl in (model, model2):
        mdl.eval()                                                                                 # evaluate.py:289
        with torch.no_grad():
            gen_e = torch.Generator().manual_seed(5)
            rows = [dict(_news(gen_e, attrs), id=f"N{i}") for i in range(60)]
            news2vector = {}
            for lo in range(0, 60, 16):                                                            # evaluate.py:193-204
                mb = default_collate(rows[lo:lo + 16])
                vec = mdl.get_news_vector(mb)
                for nid, v in zip(mb["id"], vec):
                    news2vector.setdefault(nid, v)
            dim = next(iter(news2vector.values())).shape[0]
            news2vector["PADDED_NEWS"] = torch.zeros(dim, device=dev)                             # evaluate.py:205
            users = []
            for u in range(5):                                                                     # evaluate.py:207-230
                n = [3, 50, 0, 17, 1][u]
                hist = ["PADDED_NEWS"] * (H - n) + [f"N{(7 * u + j) % 60}" for j in range(n)]
                users.append(hist)
            slot_major = [[users[b][h] for b in range(5)] for h in range(H)]                       # what default_collate yields
            clicked = torch.stack([torch.stack([news2vector[x] for x in news_list], dim=0) for news_list in slot_major],
                                  dim=0).transpose(0, 1)  # (B, H, dim) view of an (H, B, dim) stack: NON-contiguous, evaluate.py:220-224
            assert not clicked.is_contiguous()
            if name == "LSTUR":
                uv = mdl.get_user_vector(torch.tensor([3, 0, 9, 1, 2]), torch.tensor([3, 50, 0, 17, 1]), clicked)
            else:
                uv = mdl.get_user_vector(clicked)
            preds = []
            for u in range(5):                                                                     # evaluate.py:245-260
                cand = torch.stack([news2vector[f"N{(3 * u + j) % 60}"] for j in range(2 + u)], dim=0)
                p = mdl.get_prediction(cand, uv[u])
                preds.append(p.tolist())
                assert len(preds[-1]) == 2 + u
            outs.append((torch.stack([news2vector[f"N{i}"] for i in range(60)]).cpu(), uv.cpu(), preds))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1]) and outs[0][2] == outs[1][2]
    assert bool(torch.isfinite(outs[0][0]).all()) and bool(torch.isfinite(outs[0][1]).all())
