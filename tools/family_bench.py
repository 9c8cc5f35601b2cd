"""One training step (forward + backward, train mode) of every model family of the drop-in at MIND shapes
(batch 512, 1+K = 5 candidates, history 50, title 20 / abstract 50 tokens), timed with CUDA events on device-resident
inputs.  A coverage measurement next to bench.py (which is the contract benchmark on NRMS).

    python tools/family_bench.py [batch]
"""
import importlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "news-recommendation_b200", "src"))

import torch  # noqa: E402

import config as cfgmod  # noqa: E402
import newsrec_b200  # noqa: E402
from newsrec_b200 import ddp  # noqa: E402

B = int(sys.argv[1]) if len(sys.argv) > 1 else 512
dev = torch.device("cuda", 0)
C, H, T, TA = 5, 50, 20, 50


def slots(n, seed, cfg, want):
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n):
        d = {}
        if "title" in want:
            d["title"] = torch.randint(1, cfg.num_words, (B, T), generator=g).to(dev)
        if "title_entities" in want:  # MIND-like: most tokens carry no entity (id 0)
            ents = torch.randint(1, cfg.num_entities, (B, T), generator=g)
            d["title_entities"] = (ents * (torch.rand((B, T), generator=g) < 0.25)).to(dev)
        if "abstract" in want:
            d["abstract"] = torch.randint(1, cfg.num_words, (B, TA), generator=g).to(dev)
        if "category" in want:
            d["category"] = torch.randint(1, cfg.num_categories, (B,), generator=g).to(dev)
            d["subcategory"] = torch.randint(1, cfg.num_categories, (B,), generator=g).to(dev)
        out.append(d)
    return out


CASES = [
    ("NRMS", {}, ("title",)),
    ("NAML", {}, ("title", "abstract", "category")),
    ("TANR", {}, ("title", "category")),
    ("LSTUR", {"long_short_term_method": "ini"}, ("title", "category")),
    ("LSTUR", {"long_short_term_method": "con"}, ("title", "category")),
    ("Exp1", {}, ("title", "category")),
    ("HiFiArk", {}, ("title",)),
    ("DKN", {}, ("title", "title_entities")),
]
# weight of the second element of a tuple output in the training loss, per family (reference train.py)
AUX_LOSS_WEIGHT = {"TANR": "topic_classification_loss_weight", "HiFiArk": "regularizer_loss_weight"}
label = torch.zeros(B, dtype=torch.long, device=dev)
res = {}
try:  # the card and its power limit belong beside every number of this run
    card = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    card = torch.cuda.get_device_name(dev) + ", power limit unknown"
print("card:", card, flush=True)
for name, over, want in CASES:
    cfg = type("Cfg", (getattr(cfgmod, name + "Config"),), over)
    model = getattr(importlib.import_module("model." + name), name)(cfg).to(dev)
    model.train()
    grads = ddp.FlatGradients(model.parameters(), 1)
    cand, clicked = slots(C, 1, cfg, want), slots(H, 2, cfg, want)
    extra = ()
    if name == "LSTUR":
        user = torch.randint(1, cfg.num_users, (B,)).to(dev)
        length = torch.randint(1, H + 1, (B,))
        extra = (user, length)

    def step():
        grads.zero()
        out = model(*extra, cand, clicked)
        if isinstance(out, tuple):  # TANR: (click logits, topic loss); Hi-Fi Ark: (click logits, regulariser)
            loss = torch.nn.functional.cross_entropy(out[0], label) + getattr(cfg, AUX_LOSS_WEIGHT[name]) * out[1]
        else:
            loss = torch.nn.functional.cross_entropy(out, label)
        loss.backward()

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    l0 = newsrec_b200.launch_count()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 5
    key = name + ("/" + over["long_short_term_method"] if over else "")
    res[key] = {"ms_per_step": round(ms, 3), "impressions_per_s": round(B / ms * 1e3), "launches_per_step": (newsrec_b200.launch_count() - l0) // 5}
    # Hi-Fi Ark: the kernels after the news encoder (the news encoder is TANR's: compare the two step times); DKN: all of them
    kernel_keys = {"HiFiArk": ("archive",), "DKN": ("kcnn", "dkn", "archive")}.get(name)
    if kernel_keys:
        newsrec_b200.load_library().nr_profile_enable(1)
        step()
        torch.cuda.synchronize()
        res[key]["kernels_ms"] = {k: round(v[1], 4) for k, v in newsrec_b200.profile_report().items() if k.startswith(kernel_keys)}
        newsrec_b200.load_library().nr_profile_enable(0)
    print(key, res[key], flush=True)
    del model, grads
    torch.cuda.empty_cache()
print(json.dumps({"batch": B, "card": card, "families": res}))
