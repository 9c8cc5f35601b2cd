"""MMR re-ranking without a GPU: the fp64 reference (tests/mmr_ref.py) and its path verifier on hand-made cases; every
refusal of ops.top_k_scores(..., mmr_lambda=, mmr_depth=), recommend() and the CLI raised before a device is needed; the raw
nr_mmr_rerank refusing null or out-of-range arguments with -1 and a message, launching nothing; its ctypes row."""
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch

import mmr_ref as M
from newsrec_b200 import SIGNATURES, NewsrecError
from newsrec_b200 import ops
from newsrec_b200 import recommend as R

HEADER = "id\tcategory\tsubcategory\ttitle\tabstract\ttitle_entities\tabstract_entities\n"


def _one(news, rows, scores, k, lam):
    idx, sc = M.mmr_fp64(np.asarray(news, np.float32), np.array([rows]), np.array([scores], np.float32), k, lam)
    return idx[0].tolist(), sc[0]


# ---- the reference and the verifier ----

def test_lambda_one_is_the_shortlist_order():
    rng = np.random.default_rng(0)
    news = rng.standard_normal((20, 5)).astype(np.float32)
    rows = [7, 3, 12, 0, 5, 9, 1]
    scores = np.sort(rng.standard_normal(7).astype(np.float32))[::-1]
    scores[2] = scores[3]  # a tie keeps the shortlist order
    idx, sc = _one(news, rows, scores, 5, 1.0)
    assert idx == rows[:5] and sc.tolist() == scores[:5].tolist()
    idx, _ = _one(news, rows + [-1, 4], list(scores) + [-np.inf, 0.0], 9, 1.0)  # entries after the first -1 are ignored
    assert idx == rows + [-1, -1]


def test_lambda_zero_takes_the_top_one_first_then_the_least_similar():
    news = np.array([[1, 0], [1, 0.01], [0, 1], [-1, 0]], np.float32)
    idx, _ = _one(news, [0, 1, 2, 3], [4, 3, 2, 1], 4, 0.0)
    # obj is 0 for all at t = 0: the lower position; then the most dissimilar to {0} (cosine -1), then to {0, 3}
    assert idx == [0, 3, 2, 1]


def test_exact_duplicates_are_pushed_down():
    news = np.array([[1, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1], [0, 1, 1]], np.float32)
    rows, scores = [0, 1, 2, 3, 4], [1.0, 1.0, 0.9, 0.6, 0.0]
    assert _one(news, rows, scores, 3, 0.5)[0] == [0, 2, 3]  # the duplicate row 1 (cosine 1 to row 0) waits
    assert _one(news, rows, scores, 5, 0.5)[0] == [0, 2, 3, 1, 4]
    assert _one(news, rows, scores, 5, 1.0)[0] == rows


def test_equal_objectives_go_to_the_lower_position():
    news = np.eye(4, dtype=np.float32)  # orthogonal: sim 0, obj = lam rel
    idx, _ = _one(news, [3, 1, 2, 0], [2.0, 1.0, 1.0, 1.0], 4, 0.7)
    assert idx == [3, 1, 2, 0]
    idx, _ = _one(news, [3, 1, 2, 0], [1.0, 1.0, 1.0, 1.0], 4, 0.0)
    assert idx == [3, 1, 2, 0]


def test_zero_vectors_have_similarity_zero():
    news = np.array([[1, 1], [0, 0], [1, 1.001], [0, 0]], np.float32)
    rel, cos = M._user_terms(news, [0, 1, 2, 3], [3, 2, 1, 0])
    assert cos[1].tolist() == [0, 0, 0, 0] and cos[:, 3].tolist() == [0, 0, 0, 0] and cos[0, 2] > 0.99
    idx, _ = _one(news, [0, 2, 1, 3], [3, 2.9, 2, 0], 4, 0.5)
    assert idx == [0, 1, 3, 2]  # after row 0, row 2 (cosine ~1) falls behind the zero rows


def test_equal_scores_make_every_relevance_one():
    news = np.array([[1, 0], [1, 0.1], [0, 1]], np.float32)
    rel, _ = M._user_terms(news, [0, 1, 2], [0.5, 0.5, 0.5])
    assert rel.tolist() == [1, 1, 1]
    idx, _ = _one(news, [0, 1, 2], [0.5, 0.5, 0.5], 3, 0.9)
    assert idx == [0, 2, 1]
    idx, sc = _one(news, [1, -1, -1], [0.25, -np.inf, -np.inf], 3, 0.3)  # one live entry: rel 1
    assert idx == [1, -1, -1] and sc.tolist() == [0.25, -np.inf, -np.inf]


def test_the_verifier_accepts_the_reference_and_refuses_bad_paths():
    rng = np.random.default_rng(1)
    news = rng.standard_normal((50, 8)).astype(np.float32)
    sl = np.stack([rng.permutation(50)[:12] for _ in range(4)])
    scores = -np.sort(-rng.standard_normal((4, 12)).astype(np.float32), 1)
    sl[3, 9:] = -1
    scores[3, 9:] = -np.inf
    for lam in (0.0, 0.3, 1.0):
        idx, sc = M.mmr_fp64(news, sl, scores, 10, lam)
        M.verify_path(news, sl, scores, idx, sc, 10, lam)
        if lam > 0:  # the first pick swapped for the entry of least relevance (at lam = 0 every first pick is right)
            bad = idx.copy()
            worst = sl[0][int(np.argmin(scores[0]))]
            if worst in bad[0]:
                bad[0, list(bad[0]).index(worst)] = bad[0, 0]
            bad[0, 0] = worst
            bad_sc = np.array([[scores[u][list(sl[u]).index(r)] if r >= 0 else -np.inf for r in row]
                               for u, row in enumerate(bad)], np.float32)
            with pytest.raises(AssertionError):
                M.verify_path(news, sl, scores, bad, bad_sc, 10, lam)
        with pytest.raises(AssertionError):  # the score bits must be the shortlist's
            M.verify_path(news, sl, scores, idx, np.nextafter(sc, np.inf), 10, lam)
        with pytest.raises(AssertionError):  # user 3 has 9 live entries: the tenth slot is padding
            bad = idx.copy()
            bad[3, 9] = sl[3, 0]
            M.verify_path(news, sl, scores, bad, sc, 10, lam)


def test_bounds_have_the_stated_form():
    assert M.eps(300) == 2.0 ** -15 + 3 * 320 * 2.0 ** -23
    assert M.e_sim(1) == pytest.approx(2 * M.eps(1) + 2.0 ** -21, rel=1e-4)
    assert M.e_obj(300, 1.0) == 2.0 ** -20
    assert M.e_obj(300, 0.0) == M.e_sim(300) + 2.0 ** -20


# ---- refusals before the device ----

def _no_device(monkeypatch):
    def boom(*a, **k):
        raise AssertionError("device needed before the refusal")
    monkeypatch.setattr(ops, "require_cuda", boom)


BAD_LAMBDAS = (float("nan"), -0.01, 1.5, float("inf"), True, False, "0.5", None)


def test_top_k_scores_refuses_bad_mmr_requests_before_the_device(monkeypatch):
    _no_device(monkeypatch)
    users, news = torch.zeros(3, 4), torch.zeros(5, 4)
    for lam in BAD_LAMBDAS[:-1]:
        with pytest.raises(NewsrecError, match="mmr_lambda="):
            ops.top_k_scores(users, news, 2, mmr_lambda=lam)
    for depth in (1, 0, 129, 2.5, True, "8", -3):
        with pytest.raises(NewsrecError, match="mmr_depth="):
            ops.top_k_scores(users, news, 2, mmr_lambda=0.5, mmr_depth=depth)
    with pytest.raises(NewsrecError, match="needs mmr_lambda"):
        ops.top_k_scores(users, news, 2, mmr_depth=8)
    with pytest.raises(NewsrecError, match="do not combine"):
        ops.top_k_scores(users, news, 2, categories=torch.zeros(5, dtype=torch.int32), max_per_category=1, mmr_lambda=0.5)
    with pytest.raises(NewsrecError, match="do not combine"):
        ops.top_k_scores(users, news, 2, max_per_category=1, mmr_lambda=1.0)
    assert ops.mmr_request(10, 0.5, None) == (0.5, 40) and ops.mmr_request(40, 0, None) == (0.0, 128)
    assert ops.mmr_request(3, np.float32(0.25), np.int64(3)) == (0.25, 3) and ops.mmr_request(3, None, None) is None


class _Cfg:
    num_clicked_news_a_user = 4


def _fake(name):
    return type(name, (), {"config": _Cfg})()


def _split(d):
    with open(os.path.join(d, "behaviors.tsv"), "w") as f:
        f.write("1\tU1\tt\tN1\tN2-1\n")
    with open(os.path.join(d, "news_parsed.tsv"), "w") as f:
        f.write(HEADER)


def test_recommend_refuses_bad_mmr_requests_before_the_device(tmp_path, monkeypatch):
    d = str(tmp_path)
    _split(d)
    import newsrec_b200.evaluate as E

    def no_device(*a, **k):
        raise AssertionError("device work before the refusal")
    monkeypatch.setattr(R, "news_matrix", no_device)
    monkeypatch.setattr(E, "news_matrix", no_device)
    _no_device(monkeypatch)
    out = os.path.join(d, "out.tsv")
    for lam in BAD_LAMBDAS[:-1]:
        with pytest.raises(NewsrecError, match="recommend: mmr_lambda="):
            R.check_request(_fake("NRMS"), d, 10, mmr_lambda=lam)
        with pytest.raises(NewsrecError, match="recommend: mmr_lambda="):
            R.recommend(_fake("NAML"), d, out, 10, mmr_lambda=lam)
    for depth in (9, 129, 0, 12.0, False):
        with pytest.raises(NewsrecError, match="recommend: mmr_depth="):
            R.recommend(_fake("NRMS"), d, out, 10, mmr_lambda=0.5, mmr_depth=depth)
    with pytest.raises(NewsrecError, match="needs mmr_lambda"):
        R.recommend(_fake("NRMS"), d, out, 10, mmr_depth=40)
    with pytest.raises(NewsrecError, match="do not combine"):
        R.recommend(_fake("NRMS"), d, out, 10, max_per_category=2, mmr_lambda=0.5)
    for name in ("HiFiArk", "DKN"):  # the family refusal still comes first
        with pytest.raises(NewsrecError, match=f"{name} is not supported"):
            R.check_request(_fake(name), d, 10, mmr_lambda=float("nan"), mmr_depth=0)
    for lam, depth in ((0, None), (1, 10), (0.5, 128), (np.float64(0.9), np.int32(64))):
        R.check_request(_fake("NRMS"), d, 10, mmr_lambda=lam, mmr_depth=depth)
    assert not os.path.exists(out)


def test_cli_mmr_flags():
    a = R.parse_args(["--mmr-lambda", "0.5"])
    assert a.mmr_lambda == 0.5 and a.mmr_depth is None and a.max_per_category is None
    a = R.parse_args(["--mmr-lambda", "0", "--mmr-depth", "128", "--k", "100"])
    assert (a.mmr_lambda, a.mmr_depth, a.k) == (0.0, 128, 100)
    a = R.parse_args([])
    assert a.mmr_lambda is None and a.mmr_depth is None
    for bad in (["--mmr-lambda", "0.5", "--max-per-category", "2"], ["--mmr-lambda", "nan"], ["--mmr-lambda", "1.01"],
                ["--mmr-lambda", "-0.1"], ["--mmr-lambda", "inf"], ["--mmr-depth", "40"],
                ["--mmr-lambda", "0.5", "--mmr-depth", "9"], ["--mmr-lambda", "0.5", "--mmr-depth", "129"],
                ["--mmr-lambda", "x"]):
        with pytest.raises(SystemExit):
            R.parse_args(bad)


# ---- the raw entry point ----

def test_raw_entry_point_refuses_bad_arguments_without_a_device():
    import newsrec_b200
    lib = newsrec_b200.load_library()
    p, z = C.c_void_p(256), None
    #       news n   ld  D   sl_idx sl_score U  depth k  lam   idx score flag stream
    good = [p, 100, 8, 8, p, p, 4, 16, 10, 0.5, p, p, p, z]
    cases = [({0: z}, "null operand"), ({4: z}, "null operand"), ({5: z}, "null operand"), ({10: z}, "null operand"),
             ({11: z}, "null operand"), ({12: z}, "null operand"),
             ({3: 0}, "D=0"), ({3: 4097, 2: 4097}, "D=4097"), ({2: 7}, "ld_news=7"), ({1: -1}, "n_news=-1"),
             ({1: 1 << 31}, "n_news="), ({6: -1}, "n_users=-1"), ({6: 1 << 31}, "n_users="), ({7: 0}, "depth=0"),
             ({7: 129, 8: 10}, "depth=129"), ({8: 0}, "k=0"), ({8: 17}, "k=17"), ({9: float("nan")}, "lambda=nan"),
             ({9: -0.5}, "lambda=-0.5"), ({9: 1.0001}, "lambda=1"), ({9: float("inf")}, "lambda=inf")]
    for change, what in cases:
        args = list(good)
        for i, v in change.items():
            args[i] = v
        n0 = lib.nr_launch_count()
        rc = lib.nr_mmr_rerank(*args)
        msg = lib.nr_last_error().decode()
        assert rc == -1 and "nr_mmr_rerank" in msg and what in msg and lib.nr_launch_count() == n0, (change, rc, msg)
    args = list(good)
    args[6] = 0  # no user: nothing to launch, no device touched
    n0 = lib.nr_launch_count()
    assert lib.nr_mmr_rerank(*args) == 0 and lib.nr_launch_count() == n0


def test_raw_entry_point_signature():
    res, args = SIGNATURES["nr_mmr_rerank"]
    assert res is C.c_int
    assert args == [C.c_void_p, C.c_longlong, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_longlong, C.c_int, C.c_int,
                    C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    assert math.isclose(float(C.c_float(0.1).value), float(np.float32(0.1)))  # lambda reaches the kernel as fp32
