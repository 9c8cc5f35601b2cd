"""Shared by the device-feed tests: the golden fixture (oracle/make_golden_feed.py), each family's config and the
collated CPU batch of a loader item list in the golden format."""
import os

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, "tests", "golden", "feed")
BEHAVIORS = os.path.join(FIXTURE, "behaviors_parsed.tsv")
NEWS = os.path.join(FIXTURE, "news_parsed.tsv")
FAMILIES = ("NRMS", "NAML", "LSTUR", "TANR", "Exp1", "HiFiArk", "DKN")


def golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "feed.npz"))


def family_config(fam, **over):
    import config as cfgmod
    base = getattr(cfgmod, f"{fam}Config")
    return type(f"{fam}FeedConfig", (base,), over) if over else base


def collated_arrays(batch, cfg):
    """A default_collate'd minibatch as the golden arrays of one family (slots stacked on the first axis)."""
    out = {}
    for key in ("clicked_news", "candidate_news"):
        for attr in cfg.dataset_attributes["news"]:
            out[f"{key}.{attr}"] = torch.stack([slot[attr] for slot in batch[key]]).cpu().numpy()
    out["clicked"] = torch.stack(list(batch["clicked"])).cpu().numpy()
    for rec in cfg.dataset_attributes["record"]:
        out[rec] = batch[rec].cpu().numpy()
    return out


def golden_arrays(g, fam):
    return {k[len(fam) + 1:]: g[k] for k in g.files if k.startswith(fam + ".") and k != fam + ".order"}
