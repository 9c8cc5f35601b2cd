"""Test-set predictions on the H100: nr_impression_ranks against the stable-argsort restatement (tests/prediction_ref.py),
the ranks against nr_impression_metrics' place, the device text against Python's formatting, then newsrec_b200.predict end
to end for NRMS (dot scorer), LSTUR (user ids and lengths), Hi-Fi Ark (archives) and DKN (history rows) against a restated
reference loop (one get_prediction per impression, then a stable argsort), independent of the chunk size, and the CLI."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import gpu_checks as G
import prediction_ref as PR
import test_gpu_evaluate as TE

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def _ranks(scores, offsets, flag=None):
    from newsrec_b200.ops import impression_ranks
    return impression_ranks(torch.from_numpy(np.asarray(scores, np.float32)), torch.from_numpy(np.asarray(offsets, np.int64)),
                            flag)


def _text(ids, ranks, offsets):
    from newsrec_b200.ops import prediction_text
    return prediction_text(torch.from_numpy(np.asarray(ids, np.int64)), torch.from_numpy(np.asarray(ranks, np.int32)),
                           torch.from_numpy(np.asarray(offsets, np.int64))).cpu().numpy().tobytes()


def _offsets(lens):
    return np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)


def _scores(rng, n, kind):
    if kind == "normal":
        return rng.standard_normal(n).astype(np.float32)
    if kind == "ties":
        return (rng.integers(-3, 4, n) * 0.25).astype(np.float32)
    if kind == "zeros":  # -0 / +0 and subnormals of both signs, which fp32 compares under flush-to-zero would merge
        return rng.choice(np.array([-0.0, 0.0, 1e-45, -1e-45, 3e-39, -3e-39, 1.0], np.float32), n)
    return np.full(n, 0.5, np.float32)


@pytest.mark.parametrize("n", [1, 31, 32, 33, 511, 512, 513, 1500])
def test_ranks_equal_the_stable_argsort(n):
    rng = np.random.default_rng(n)
    kinds = ["normal", "ties", "zeros", "equal"]
    lens = [n] * 4 * len(kinds)
    scores = np.concatenate([_scores(rng, n, k) for k in kinds for _ in range(4)])
    offsets = _offsets(lens)
    got = _ranks(scores, offsets).cpu().numpy()
    np.testing.assert_array_equal(got, PR.impression_ranks(scores, offsets))
    for a, b in zip(offsets[:-1], offsets[1:]):
        np.testing.assert_array_equal(np.sort(got[a:b]), np.arange(1, b - a + 1))


def test_ranks_with_more_impressions_than_resident_warps():
    rng = np.random.default_rng(11)
    lens = rng.integers(1, 80, 40_000)            # 148 * 16 blocks of 8 warps hold 18,944: every warp loops
    lens[::997] = 700                             # and some impressions span two shared-memory chunks
    offsets = _offsets(lens)
    scores = (rng.integers(-6, 7, offsets[-1]) * 0.125).astype(np.float32)
    scores[scores == 0] = np.where(rng.random(int((scores == 0).sum())) < 0.5, np.float32(-0.0), np.float32(0.0))
    got = _ranks(scores, offsets).cpu().numpy()
    np.testing.assert_array_equal(got, PR.impression_ranks(scores, offsets))


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf])
def test_a_non_finite_score_sets_the_flag(bad):
    offsets = _offsets([3, 4, 2])
    scores = np.array([0.1, 0.2, 0.3, 0.4, bad, 0.0, 1.0, 2.0, 1.0], np.float32)
    with pytest.raises(ValueError, match="non-finite"):
        _ranks(scores, offsets)
    flag = torch.zeros(1, dtype=torch.int32, device=DEV)
    got = _ranks(scores, offsets, flag).cpu().numpy()
    assert int(flag.item()) == 1
    np.testing.assert_array_equal(got, [3, 2, 1, 0, 0, 0, 0, 1, 2])  # the bad impression's ranks are 0, the others hold


def test_ranks_take_the_place_of_the_metrics():
    from newsrec_b200.ops import impression_metrics
    rng = np.random.default_rng(3)
    lens = list(rng.integers(1, 300, 20_000)) + [513, 1500]
    offsets = _offsets(lens)
    n = int(offsets[-1])
    scores = (rng.integers(-4, 5, n) * 0.25).astype(np.float32)
    labels = (rng.random(n) < 0.2).astype(np.uint8)
    ranks = _ranks(scores, offsets).cpu().numpy()
    m = impression_metrics(torch.from_numpy(scores), torch.from_numpy(labels), torch.from_numpy(offsets)).cpu().numpy()
    mrr = np.array([np.mean(1.0 / ranks[a:b][labels[a:b] == 1]) if labels[a:b].any() else np.nan
                    for a, b in zip(offsets[:-1], offsets[1:])])
    np.testing.assert_array_equal(np.isnan(mrr), np.isnan(m[:, 1]))
    ok = ~np.isnan(mrr)
    assert ok.sum() > 15_000 and np.abs(mrr[ok] - m[ok, 1]).max() <= 1e-12


def test_text_bytes_equal_python_formatting():
    rng = np.random.default_rng(4)
    lens = [1, 1, 9, 10, 11, 99, 100, 101, 1000, 1, 37]  # ranks crossing 9 -> 10, 99 -> 100, 999 -> 1000
    ids = [0, 9, 10, 1 << 40, 99, 100, (1 << 63) - 1, 7, 123456789, 1, 10 ** 12]
    offsets = _offsets(lens)
    ranks = np.concatenate([rng.permutation(k) + 1 for k in lens]).astype(np.int32)
    assert _text(ids, ranks, offsets) == PR.prediction_text(ids, ranks, offsets)
    # many impressions (more than resident warps), ids and ranks from the ranks kernel
    lens = rng.integers(1, 300, 30_000)
    offsets = _offsets(lens)
    ids = rng.integers(0, 1 << 62, len(lens))
    scores = rng.standard_normal(int(offsets[-1])).astype(np.float32)
    ranks = _ranks(scores, offsets).cpu().numpy()
    assert _text(ids, ranks, offsets) == PR.prediction_text(ids.tolist(), ranks, offsets)
    assert _text([], np.zeros(0, np.int32), [0]) == b""


# ------------------------------------------------------------------------------------------------------------------------
# end to end
# ------------------------------------------------------------------------------------------------------------------------
FAMILIES = ["NRMS", "LSTUR", "HiFiArk", "DKN"]


def _model(name):
    import config
    torch.manual_seed(0)
    if name in ("NRMS", "LSTUR"):
        model, cfg = G.build_model({"NRMS": "nrms", "LSTUR": "lstur_ini"}[name], V=TE.V, ncat=TE.NCAT, nusers=TE.NUSERS, H=TE.H)
        cfg.batch_size = 2                    # batches of 32 news / users: several of each
    elif name == "HiFiArk":
        from model.HiFiArk import HiFiArk
        model = HiFiArk(type("Cfg", (config.HiFiArkConfig,), dict(num_words=TE.V, num_clicked_news_a_user=TE.H, batch_size=2))).to(DEV)
    else:
        from model.DKN import DKN
        cfg = type("Cfg", (config.DKNConfig,), dict(num_words=TE.V, num_entities=30, num_clicked_news_a_user=TE.H, batch_size=2))
        model = DKN(cfg).to(DEV)
        with torch.no_grad():  # entity rows non-trivial although the synthetic titles carry no entity
            model.kcnn.entity_embedding.weight[0].uniform_(-1, 1)
    return model.eval()


def _strip_labels(src, dst):
    os.makedirs(dst, exist_ok=True)
    for f in ("news_parsed.tsv", "user2int.tsv"):
        with open(os.path.join(src, f)) as a, open(os.path.join(dst, f), "w") as b:
            b.write(a.read())
    with open(os.path.join(src, "behaviors.tsv")) as a, open(os.path.join(dst, "behaviors.tsv"), "w") as b:
        for ln in a:
            r = ln.rstrip("\n").split("\t")
            r[4] = " ".join(x.split("-")[0] for x in r[4].split())
            b.write("\t".join(r) + "\n")


def _reference_ranks(model, d):
    """One get_prediction per impression (src/evaluate.py:245-265) on the news matrix and each impression's first-wins
    history, then the ranks of a stable argsort.  Also returns, per impression, whether two restated scores lie within
    1e-5 relative of each other (an ulp-level difference could then swap them)."""
    from newsrec_b200 import evaluate as E
    H = model.config.num_clicked_news_a_user
    lstur = type(model).__name__ == "LSTUR"
    with torch.no_grad():
        index, matrix = E.news_matrix(model, d)
        t = E.build_tables(d, index, H, 10 ** 9, os.path.join(d, "user2int.tsv"))
        out, near = [], []
        for s in range(len(t.seg_user)):
            u = t.seg_user[s]
            hist = matrix[torch.from_numpy(t.history[u])].unsqueeze(0)
            uv = (model.get_user_vector(torch.tensor([t.user[u]]), torch.tensor([t.history_length[u]]), hist) if lstur
                  else model.get_user_vector(hist))[0]
            cand = matrix[torch.from_numpy(t.cand[t.seg_offsets[s]:t.seg_offsets[s + 1]])]
            y = model.get_prediction(cand, uv).double().cpu().numpy().reshape(-1)
            out.append(PR.single_ranks(y))
            p = np.sort(y)
            near.append(len(p) > 1 and not (np.diff(p) > 1e-5 * np.maximum(np.abs(p[1:]), np.abs(p[:-1]))).all())
    return t, out, np.array(near)


def _read_lines(path):
    ids, ranks = [], []
    for ln in open(path, "rb").read().decode().splitlines():
        i, r = ln.split(" ", 1)
        assert r[0] == "[" and r[-1] == "]", ln
        ids.append(int(i))
        ranks.append(np.array([int(x) for x in r[1:-1].split(",")]))
    return ids, ranks


@pytest.mark.parametrize("name", FAMILIES)
def test_prediction_file_matches_the_reference_loop(name, tmp_path):
    from newsrec_b200 import evaluate as E
    from newsrec_b200.predict import predict
    lab, test = str(tmp_path / "val"), str(tmp_path / "test")
    os.makedirs(lab)
    TE._write_validation_dir(lab)
    _strip_labels(lab, test)
    model = _model(name)
    u2i = os.path.join(test, "user2int.tsv")
    files = {}
    for chunk in (1, 7, 10 ** 9):
        files[chunk] = str(tmp_path / f"prediction_{chunk}.txt")
        assert predict(model, test, files[chunk], user2int_path=u2i, chunk_impressions=chunk) == 60
        assert not os.path.exists(files[chunk] + ".partial")
    data = {k: open(v, "rb").read() for k, v in files.items()}
    assert data[1] == data[7] == data[10 ** 9]
    ids, ranks = _read_lines(files[1])
    t, ref, near = _reference_ranks(model, lab)
    assert ids == list(range(1, 61)) and len(ref) == 60
    assert near.sum() <= 3, near.sum()
    for s in np.flatnonzero(~near):
        np.testing.assert_array_equal(ranks[s], ref[s], err_msg=f"impression {s + 1}")
    for r in ranks:
        np.testing.assert_array_equal(np.sort(r), np.arange(1, len(r) + 1))
    # with the labels back: MRR from the file is evaluate()'s MRR
    got = E.evaluate(model, lab, 4, user2int_path=u2i)
    offs, y = t.seg_offsets, t.labels
    mrr = [np.mean(1.0 / ranks[s][y[offs[s]:offs[s + 1]] == 1]) if y[offs[s]:offs[s + 1]].any() else np.nan for s in range(60)]
    assert abs(np.nanmean(mrr) - got[1]) <= 1e-12, (np.nanmean(mrr), got[1])


def test_a_non_finite_score_raises_and_leaves_no_file(tmp_path, monkeypatch):
    from newsrec_b200 import predict as P
    d = str(tmp_path)
    TE._write_validation_dir(d)
    model = _model("NRMS")
    orig, calls = P.impression_scores, []

    def poisoned(*a, **k):  # the third chunk's last candidate (impressions 33..48)
        s = orig(*a, **k)
        calls.append(1)
        if len(calls) == 3:
            s[-1] = float("nan")
        return s

    monkeypatch.setattr(P, "impression_scores", poisoned)
    out = str(tmp_path / "prediction.txt")
    with pytest.raises(ValueError, match=r"impression 48 \(behaviors.tsv line 48\) has a non-finite score"):
        P.predict(model, d, out, user2int_path=os.path.join(d, "user2int.tsv"), chunk_impressions=16)
    assert not os.path.exists(out) and not os.path.exists(out + ".partial")


def test_cli_writes_the_same_file(tmp_path):
    from newsrec_b200.predict import predict
    test = str(tmp_path / "test")
    os.makedirs(test)
    TE._write_validation_dir(test)
    model = _model("NRMS")
    u2i = os.path.join(test, "user2int.tsv")
    ref = str(tmp_path / "in_process.txt")
    predict(model, test, ref, user2int_path=u2i)
    ck = tmp_path / "checkpoint" / "NRMS"
    ck.mkdir(parents=True)
    state = {"model_state_dict": model.state_dict(), "optimizer_state_dict": {}, "step": 5, "early_stop_value": -np.float64(0.5)}
    torch.save(state, str(ck / "ckpt-5.pth"))
    torch.save({**state, "model_state_dict": {}}, str(ck / "ckpt-2.pth"))  # an older checkpoint: not loaded
    src = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "news-recommendation_b200", "src")
    env = dict(os.environ, MODEL_NAME="NRMS", PYTHONPATH=os.pathsep.join([src, os.environ.get("PYTHONPATH", "")]))
    cfg = model.config
    knobs = [f"--set={k}={getattr(cfg, k)!r}" for k in ("num_words", "num_categories", "num_users", "num_clicked_news_a_user",
                                                       "dropout_probability", "precision", "batch_size")]
    out = str(tmp_path / "cli.txt")
    res = subprocess.run([sys.executable, "-m", "newsrec_b200.predict", "--directory", test, "--out", out, "--user2int", u2i,
                          *knobs], cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stdout + res.stderr
    assert "ckpt-5.pth" in res.stdout and "60 impressions" in res.stdout
    assert open(out, "rb").read() == open(ref, "rb").read()
