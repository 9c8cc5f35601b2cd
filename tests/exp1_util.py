"""Helpers of the Exp1 tests: the golden case's parameters and inputs for the oracle (oracle/exp1_oracle.py) and the drop-in."""
import torch

import exp1_oracle as E
import newsrec_oracle as O
from golden_util import NCAT, V, load_case

H = 6  # num_clicked_news_a_user of the golden case (oracle/make_golden.py)


def exp1_params(g, dtype=torch.float32, requires_grad=True):
    """The golden case's state_dict as leaf tensors; the shared category table is ONE leaf under both element-encoder keys."""
    sd = E.exp1_state_dict(V, NCAT, H, int(g["seed"]))
    out, seen = {}, {}
    for k, v in sd.items():
        if id(v) in seen:
            out[k] = out[seen[id(v)]]
            continue
        seen[id(v)] = k
        out[k] = v.to(dtype).clone().requires_grad_(requires_grad)
    return out


def exp1_fields(g):
    """({name: (B, C, ...)}, {name: (B, H, ...)}) of the golden case."""
    t = lambda k: torch.from_numpy(g[k])
    names = ("title", "category", "subcategory")
    return {n: t("cand_" + n) for n in names}, {n: t("clicked_" + n) for n in names}


def oracle_logits(g, p, contract=O.EXACT, drop=None):
    cand, clicked = exp1_fields(g)
    return E.exp1_forward(cand, clicked, p, 15, contract, drop)


def slot_lists(g):
    """The reference DataLoader's slot-major lists of per-slot dicts."""
    cand, clicked = exp1_fields(g)
    mk = lambda d: [{k: v[:, j].contiguous() for k, v in d.items()} for j in range(d["title"].shape[1])]
    return mk(cand), mk(clicked)


def golden_grad_key(k, g):
    """The golden file names the shared category table by its first registration in the reference (a set order)."""
    if "gsum:" + k in g:
        return k
    for a, b in (("category", "subcategory"), ("subcategory", "category")):
        kk = k.replace(f".{a}.", f".{b}.")
        if "gsum:" + kk in g:
            return kk
    return None


def load():
    return load_case("exp1")


def relerr(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / max(b.norm().item(), 1e-30))
