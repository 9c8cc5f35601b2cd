"""Device evaluator on the H100: nr_impression_metrics against the live reference's values (golden) and the NumPy oracle at
scale, then newsrec_b200.evaluate.evaluate for every model family, stage by stage, against the reference evaluator's call
sequence restated around the drop-in model (as tests/test_gpu_integration.py does: the reference's drivers do not travel
to the GPU machine).  Each step of the restatement cites the line it mirrors in src/evaluate.py."""
import os
from ast import literal_eval

import numpy as np
import pytest
import torch
from torch.utils.data import default_collate

import gpu_checks as G
import ranking_metrics as R

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def _kernel(scores, labels, offsets):
    from newsrec_b200.ops import impression_metrics
    return impression_metrics(torch.from_numpy(np.asarray(scores, np.float32)), torch.from_numpy(np.asarray(labels, np.uint8)),
                              torch.from_numpy(np.asarray(offsets, np.int64))).cpu().numpy()


def _close(got, ref, tol=1e-12):
    np.testing.assert_array_equal(np.isnan(got), np.isnan(ref))
    d = np.abs(np.where(np.isnan(ref), 0.0, got - ref))
    assert d.max() <= tol, (d.max(), np.unravel_index(d.argmax(), d.shape))


def test_kernel_matches_the_reference_golden(golden_dir):
    g = np.load(os.path.join(golden_dir, "eval_metrics.npz"))
    got = _kernel(g["scores"], g["labels"], g["offsets"])
    ref, cross = g["ref"].copy(), g["cross_tie"]
    # where tied candidates carry different labels the reference's MRR / nDCG come from NumPy's unstable sort: compare
    # those with the stable rule the kernel pins (the oracle), AUC with the reference itself
    ref[cross, 1:] = R.impression_metrics(g["scores"], g["labels"], g["offsets"])[cross, 1:]
    _close(got, ref)


def test_kernel_matches_the_oracle_at_scale():
    rng = np.random.default_rng(7)
    lens = list(rng.integers(1, 401, 100_000)) + [2000, 2047, 3001, 4500]
    offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    n = int(offsets[-1])
    scores = rng.integers(-4, 5, n).astype(np.float32) * np.float32(0.25)    # a small integer set: ties everywhere
    scores[rng.random(n) < 2e-6] = np.nan
    scores[rng.random(n) < 2e-6] = -np.inf
    scores[scores == 0] = np.where(rng.random(int((scores == 0).sum())) < 0.5, np.float32(-0.0), np.float32(0.0))
    p_pos = np.repeat(rng.choice([0.0, 0.05, 0.3, 1.0], len(lens), p=[0.02, 0.6, 0.36, 0.02]), lens)
    labels = (rng.random(n) < p_pos).astype(np.uint8)
    got = _kernel(scores, labels, offsets)
    ref = R.impression_metrics(scores, labels, offsets)
    assert np.isnan(ref[:, 0]).sum() > 100 and (~np.isnan(ref)).all(1).sum() > 90_000
    _close(got, ref)


def test_kernel_rejects_labels_other_than_0_1():
    with pytest.raises(ValueError):
        _kernel([0.1, 0.2, 0.3], [1, 2, 0], [0, 3])
    assert _kernel([], [], [0]).shape == (0, 4)


# ------------------------------------------------------------------------------------------------------------------------
# end to end
# ------------------------------------------------------------------------------------------------------------------------
V, NCAT, NUSERS, H, T, TA = 300, 12, 40, 50, 20, 50
N_NEWS = 150
CASES = {"NRMS": "nrms", "NAML": "naml", "LSTUR": "lstur_ini", "TANR": "tanr"}


def _write_validation_dir(d, seed=3):
    """news_parsed.tsv (tools/make_synth_mind.py's columns), raw-format behaviors.tsv, user2int.tsv."""
    rng = np.random.default_rng(seed)
    news = [f"N{i}" for i in range(N_NEWS)]

    def padded(n, length):
        return [int(x) for x in rng.integers(1, V, n)] + [0] * (length - n)

    with open(os.path.join(d, "news_parsed.tsv"), "w") as f:
        f.write("id\tcategory\tsubcategory\ttitle\tabstract\ttitle_entities\tabstract_entities\n")
        for nid in news:
            f.write(f"{nid}\t{rng.integers(1, NCAT)}\t{rng.integers(1, NCAT)}\t{padded(int(rng.integers(5, T + 1)), T)}\t"
                    f"{padded(int(rng.integers(10, TA + 1)), TA)}\t{[0] * T}\t{[0] * TA}\n")
    hists = [" ".join(rng.choice(news, int(k), replace=True)) for k in (3, 60, 0, 17, 1, 75, 50, 8, 0, 22)]
    users = [f"U{i}" for i in range(12)]
    rows = []
    for i in range(60):
        u = users[i % len(users)]
        h = hists[(i * 7) % len(hists)]
        if i in (5, 6):
            u, h = ["U0", "U11"][i - 5], hists[1]                  # the same history under two users
        k = int(rng.integers(2, 15))
        cand = rng.choice(news, k, replace=False)                  # distinct candidates within an impression
        lab = (rng.random(k) < 0.3).astype(int)
        if i % 9 == 4:
            lab[:] = 1                                             # no negative
        elif i % 9 == 7:
            lab[:] = 0                                             # no positive
        elif lab.sum() == 0:
            lab[0] = 1
        rows.append(f"{i + 1}\t{u}\t11/15/2019 8:55:22 AM\t{h}\t{' '.join(f'{c}-{y}' for c, y in zip(cand, lab))}\n")
    with open(os.path.join(d, "behaviors.tsv"), "w") as f:
        f.writelines(rows)
    with open(os.path.join(d, "user2int.tsv"), "w") as f:
        f.write("user\tint\n" + "".join(f"U{i}\t{i + 1}\n" for i in range(10)))  # U10, U11 unknown -> 0


def _reference_loop(model, d, attrs, max_count):
    """src/evaluate.py:171-265 restated around the model: (news2vector, user2vector, [(y_true, y_pred)])."""
    import pandas as pd
    lstur = type(model).__name__ == "LSTUR"
    bs = model.config.batch_size * 16
    news = pd.read_table(os.path.join(d, "news_parsed.tsv"), usecols=["id"] + attrs,
                         converters={a: literal_eval for a in set(attrs) & {"title", "abstract"}})
    items = [{"id": r["id"], **{a: torch.tensor(r[a]) for a in attrs}} for r in news.to_dict("records")]   # :54-76
    news2vector = {}
    for lo in range(0, len(items), bs):                                                                       # :193-204
        mb = default_collate(items[lo:lo + bs])
        vec = model.get_news_vector(mb)
        for nid, v in zip(mb["id"], vec):
            news2vector.setdefault(nid, v)
    news2vector["PADDED_NEWS"] = torch.zeros(next(iter(news2vector.values())).size())                        # :205-206
    beh = [ln.rstrip("\n").split("\t") for ln in open(os.path.join(d, "behaviors.tsv"))]
    user2int = dict(ln.rstrip("\n").split("\t") for ln in list(open(os.path.join(d, "user2int.tsv")))[1:])
    seen, urows = set(), []
    for r in beh:                                                                                             # :79-121
        key = (r[1], r[3] or " ")
        if key not in seen:
            seen.add(key)
            hs = key[1].split()[:H]
            urows.append({"user": int(user2int.get(r[1], 0)), "clicked_news_string": key[1],
                          "clicked_news": ["PADDED_NEWS"] * (H - len(hs)) + hs, "clicked_news_length": len(hs)})
    user2vector = {}
    for lo in range(0, len(urows), bs):                                                                       # :216-230
        mb = default_collate(urows[lo:lo + bs])
        cnv = torch.stack([torch.stack([news2vector[x].to(DEV) for x in news_list], dim=0)
                           for news_list in mb["clicked_news"]], dim=0).transpose(0, 1)
        uv = model.get_user_vector(mb["user"], mb["clicked_news_length"], cnv) if lstur else model.get_user_vector(cnv)
        for s, v in zip(mb["clicked_news_string"], uv):
            user2vector.setdefault(s, v)
    tasks = []
    count = 0
    for r in beh:                                                                                             # :243-265
        count += 1
        if count == max_count:
            break
        imp = r[4].split()
        cand = torch.stack([news2vector[x.split("-")[0]] for x in imp], dim=0)
        y_pred = model.get_prediction(cand, user2vector[r[3] or " "]).tolist()
        tasks.append(([int(x.split("-")[1]) for x in imp], y_pred))
    return news2vector, user2vector, tasks


def _rel(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


@pytest.mark.parametrize("name", ["NRMS", "NAML", "LSTUR", "TANR"])
def test_device_evaluator_matches_the_reference_loop(name, tmp_path):
    from newsrec_b200 import evaluate as E
    d = str(tmp_path)
    _write_validation_dir(d)
    torch.manual_seed(0)
    model, cfg = G.build_model(CASES[name], V=V, ncat=NCAT, nusers=NUSERS, H=H)
    cfg.batch_size = 2                        # batches of 32 news / users: several of each
    attrs = list(cfg.dataset_attributes["news"])
    model.eval()
    u2i = os.path.join(d, "user2int.tsv")
    max_count = 10 ** 9
    with torch.no_grad():
        news2vector, user2vector, tasks = _reference_loop(model, d, attrs, max_count)
        index, matrix = E.news_matrix(model, d)
        tables = E.build_tables(d, index, H, max_count, u2i)
        flag = E.new_flag(DEV)
        users = E.user_vectors(model, tables, matrix, flag)
        scores = E.impression_scores(tables, matrix, users, flag)
        torch.cuda.synchronize()
        assert int(flag.item()) == 0
    # stage 1: news matrix rows bitwise equal, pad row zero
    ids = [k for k in news2vector if k != "PADDED_NEWS"]
    assert torch.equal(matrix[[index[k] for k in ids]].cpu(), torch.stack([news2vector[k] for k in ids]).cpu())
    assert not matrix[index["PADDED_NEWS"]].any()
    # stage 2: one user vector per distinct history string
    hist_strings = list(user2vector)
    assert len(hist_strings) == len(tables.user)
    mine = users[torch.arange(len(hist_strings))]
    ref_u = torch.stack([user2vector[s] for s in hist_strings])  # first appearance order == build_tables' row order
    assert _rel(mine, ref_u) <= 1e-6, _rel(mine, ref_u)
    # stage 3: scores against per-impression get_prediction
    offs = tables.seg_offsets
    assert len(offs) - 1 == len(tasks)
    worst = 0.0
    for s, (y_true, y_pred) in enumerate(tasks):
        got = scores[offs[s]:offs[s + 1]].cpu().double()
        ref = torch.tensor(y_pred, dtype=torch.float64)
        worst = max(worst, _rel(got, ref))
        assert list(tables.labels[offs[s]:offs[s + 1]]) == y_true
        # no two restated scores of an impression within 1e-5 relative: an ulp-level rank flip cannot pass for a bug.  The
        # one exception is exact: an empty history gives NAML / TANR a zero user vector, every score is 0.0 in both paths
        p = np.sort(np.asarray(y_pred))
        if p[0] == p[-1] == 0.0:
            assert bool((got == 0).all()), (s, got)
            continue
        assert (np.diff(p) > 1e-5 * np.maximum(np.abs(p[1:]), np.abs(p[:-1]))).all(), (s, y_pred)
    assert worst <= 1e-6, worst
    assert any(sum(y) == len(y) for y, _ in tasks) and any(sum(y) == 0 for y, _ in tasks)
    # the four means against the oracle on the restated scores, and max_count = k scores exactly k - 1 impressions
    for k in (max_count, 17):
        sub = tasks[:k - 1]
        ref = np.nanmean(np.array([R.single_impression(y_pred, y_true) for y_true, y_pred in sub]), axis=0)
        got = E.evaluate(model, d, 4, k, user2int_path=u2i)
        assert all(isinstance(v, np.float64) for v in got)
        assert np.abs(np.array(got) - ref).max() <= 1e-6, (got, ref)
    assert len(E.build_tables(d, index, H, 17, u2i).seg_user) == 16
