"""Diversified recommendation on the H100: nr_topk_dot_capped / ops.top_k_scores(..., categories=, max_per_category=) and
newsrec_b200.recommend(..., max_per_category=, diversify_by=), against the walk restated on the kernel's own scores.

The contract (include/newsrec_b200.h): walk the pool without the user's exclusions in nr_topk_dot's order (score descending,
then lower row) and take a news iff fewer than m taken news share its category and fewer than k are taken.  The oracle gets
every (user, news) score bit for bit from ops.pool_ranks (the same planes and tile code as nr_topk_dot; every news is a
target of its user, 32 targets per kernel row, a row's targets neighbours in fp64 order so that the ranks it also counts
stay cheap) and runs that walk, so idx and score must be torch.equal to the kernel's.  A sanity check against fp64 uses the
bound of nr_topk_dot, e_un = (2^-15 + 3 round_up(D, 64) 2^-23) sum_i |u_i||n_i|."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import gpu_checks as G
import test_gpu_evaluate as TE
import test_gpu_recommend as TR

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
I32_MIN, I32_MAX = -2 ** 31, 2 ** 31 - 1


def kernel_scores(users, news):
    """(U, n) fp32: s(u, r) bit for bit as nr_topk_dot computes it, from ops.pool_ranks with every news a target of its user."""
    from newsrec_b200.ops import pool_ranks
    users, news = users.to(DEV).float(), news.to(DEV).float()
    U, n = users.shape[0], news.shape[0]
    if U == 0 or n == 0:
        return torch.zeros((U, n), dtype=torch.float32, device=DEV)
    P = (n + 31) // 32
    order = torch.argsort(users.double() @ news.double().T, dim=1, descending=True)  # (U, n) rows, fp64 order
    counts = np.full((U, P), 32, np.int64)
    counts[:, -1] = n - 32 * (P - 1)
    offs = np.zeros(U * P + 1, np.int64)
    offs[1:] = np.cumsum(counts.reshape(-1))
    _, score = pool_ranks(users.repeat_interleave(P, 0), news, order.reshape(-1).cpu(), offs)
    out = torch.empty((U, n), dtype=torch.float32, device=DEV)
    out.scatter_(1, order, score.view(U, n))
    return out


def host_walk(S, cat, m, k, elig=None):
    """The capped walk over the exact scores S (U, n) fp32 with keys cat (n,): (idx (U, k) int64, score (U, k) fp32)."""
    S = S.to(DEV)
    U, n = S.shape
    idx = torch.full((U, k), -1, dtype=torch.int64, device=DEV)
    sc = torch.full((U, k), float("-inf"), dtype=torch.float32, device=DEV)
    if U == 0 or n == 0:
        return idx, sc
    elig = torch.ones_like(S, dtype=torch.bool) if elig is None else elig.to(DEV)
    key = torch.where(elig, S, torch.tensor(float("-inf"), device=DEV))
    # rows ascending, then a stable descending sort: equal scores keep the lower row first (finite scores: eligible first)
    s_sorted, order = torch.sort(key, dim=1, descending=True, stable=True)
    live = torch.gather(elig, 1, order)
    c = torch.as_tensor(np.asarray(cat, np.int64), device=DEV)[order]
    cs, perm = torch.sort(c, dim=1, stable=True)  # walk order within each category
    pos = torch.arange(n, device=DEV).expand(U, n)
    start = torch.ones_like(cs, dtype=torch.bool)
    start[:, 1:] = cs[:, 1:] != cs[:, :-1]
    occ_sorted = pos - torch.where(start, pos, torch.zeros_like(pos)).cummax(dim=1).values
    occ = torch.empty_like(occ_sorted).scatter_(1, perm, occ_sorted)  # earlier entries of the same category
    keep = live & (occ < m)
    keep &= torch.cumsum(keep.int(), dim=1) <= k
    for u in range(U):
        p = torch.nonzero(keep[u]).flatten()
        idx[u, :len(p)] = order[u, p]
        sc[u, :len(p)] = s_sorted[u, p]
    return idx, sc


def _capped(users, news, k, cat, m, excl=None):
    from newsrec_b200.ops import top_k_scores
    rows, offs = TR._csr(excl) if excl is not None else (None, None)
    return top_k_scores(users, news, k, rows, offs, categories=torch.as_tensor(np.asarray(cat), dtype=torch.int32),
                        max_per_category=m)


def _elig(U, n, excl):
    elig = torch.ones((U, n), dtype=torch.bool, device=DEV)
    if excl is not None:
        for u, lst in enumerate(excl):
            if len(lst):
                elig[u, torch.as_tensor(np.asarray(lst, np.int64), device=DEV)] = False
    return elig


def _check(users, news, k, cat, m, excl=None, S=None):
    """The kernel's capped lists equal the host walk over its exact scores (S: kernel_scores(users, news) when given), obey
    the caps, and lie within the fp64 bound."""
    idx, score = _capped(users, news, k, cat, m, excl)
    U, n, D = users.shape[0], news.shape[0], users.shape[1]
    assert idx.shape == (U, k) and score.shape == (U, k)
    elig = _elig(U, n, excl)
    want_i, want_s = host_walk(kernel_scores(users, news) if S is None else S, cat, m, k, elig)
    assert torch.equal(idx.to(DEV), want_i), "idx differs from the walk over the kernel's scores"
    assert G._bits_equal(score.to(DEV), want_s), "score differs from the walk over the kernel's scores"
    live = want_i >= 0
    assert torch.equal(live, torch.arange(k, device=DEV)[None, :] < live.sum(1, keepdim=True)), "live slots first"
    r = want_i.clamp(min=0)
    assert bool(torch.gather(elig, 1, r)[live].all()), "an excluded news was returned"
    ct = torch.as_tensor(np.asarray(cat, np.int64), device=DEV)[r]
    for u in range(U):
        _, cnt = torch.unique(ct[u][live[u]], return_counts=True)
        assert cnt.numel() == 0 or int(cnt.max()) <= m, "a category over its cap"
    u64, n64 = users.double().to(DEV), news.double().to(DEV)
    s_ref = (u64[:, None, :] * n64[r]).sum(-1)
    e_ref = TR._bound_coeff(D) * (u64.abs()[:, None, :] * n64[r].abs()).sum(-1)
    assert bool(((score.to(DEV).double() - s_ref).abs() <= e_ref)[live].all()), "score bound"
    return idx, score


def _randn(seed, *shape):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


def _zipf(rng, n, n_cat, s=1.1):
    p = 1.0 / np.arange(1, n_cat + 1) ** s
    return rng.choice(n_cat, n, p=p / p.sum()).astype(np.int32)


# ---- 1. exact oracle at every shape of test_gpu_recommend ----
@pytest.mark.parametrize("U,n,D,k", TR.CASES)
def test_capped_matches_the_walk_over_the_kernel_scores(U, n, D, k):
    seed = U * 7 + n + D + k
    users, news = _randn(seed, U, D), _randn(seed + 1, n, D)
    rng = np.random.default_rng(seed)
    S = kernel_scores(users, news)
    _check(users, news, k, rng.integers(0, 17, n).astype(np.int32), 2, S=S)   # 17 categories, m = 2
    _check(users, news, k, _zipf(rng, n, 264), 1, S=S)                        # Zipf over 264, m = 1
    _check(users, news, k, rng.integers(0, 3, n), 1, S=S)                     # caps that run out when k > 3


# ---- 2. category mixes ----
MIX_U, MIX_N, MIX_D = 130, 5000, 300


def _mix_inputs(seed=11):
    return _randn(seed, MIX_U, MIX_D), _randn(seed + 1, MIX_N, MIX_D)


@pytest.mark.parametrize("k", [10, 100])
def test_category_mixes(k):
    users, news = _mix_inputs()
    rng = np.random.default_rng(k)
    S = kernel_scores(users, news)
    _check(users, news, k, rng.integers(0, 17, MIX_N), 2, S=S)            # uniform over 17
    _check(users, news, k, _zipf(rng, MIX_N, 264), 1, S=S)                 # Zipf over 264
    idx, score = _check(users, news, k, np.full(MIX_N, 5), 3, S=S)         # one category: exactly min(m, k)
    assert bool(((idx >= 0).sum(1) == min(3, k)).all())
    distinct = np.arange(MIX_N)                                       # every news its own category: the plain answer
    from newsrec_b200.ops import top_k_scores
    i0, s0 = top_k_scores(users, news, k)
    i1, s1 = _check(users, news, k, distinct, 1, S=S)
    assert torch.equal(i0, i1) and G._bits_equal(s0, s1)


@pytest.mark.parametrize("where", ["first", "last"])
def test_top_category_all_in_the_first_or_last_tiles(where):
    users, news = _mix_inputs(12)
    n, D = MIX_N, MIX_D
    g = torch.Generator().manual_seed(13)
    rows = np.arange(300) if where == "first" else np.arange(n - 300, n)
    users += 3.0                                                      # u . 1 ~ 900, far above any random news' score
    news[torch.as_tensor(rows)] = 1.0 + 0.3 * torch.randn(len(rows), D, generator=g)
    cat = np.random.default_rng(14).integers(1, 40, n)
    cat[rows] = 0                                                     # the top-scoring category, category 0
    S = kernel_scores(users, news)
    for k, m in ((10, 2), (100, 1), (128, 30)):
        idx, _ = _check(users, news, k, cat, m, S=S)
        top = torch.as_tensor(np.isin(np.arange(n), rows), device=DEV)[idx.to(DEV).clamp(min=0)] & (idx.to(DEV) >= 0)
        assert bool((top.sum(1) == m).all()), "the top category fills exactly its cap"


def test_caps_that_run_out_and_odd_keys():
    users, news = _mix_inputs(15)
    rng = np.random.default_rng(15)
    S = kernel_scores(users, news)
    three = rng.integers(0, 3, MIX_N)
    for k, m in ((10, 2), (128, 5), (100, 1)):
        idx, score = _check(users, news, k, three, m, S=S)                 # 3 categories x m < k: short lists
        assert bool(((idx >= 0).sum(1) == 3 * m).all())
        assert bool((idx[:, 3 * m:] == -1).all()) and bool((score[:, 3 * m:] == float("-inf")).all())
    keys = np.array([0, -1, -5, 7, I32_MIN, I32_MAX], np.int64)
    _check(users, news, 10, rng.choice(keys, MIX_N), 2, S=S)               # 0, negative keys and the int32 extremes
    _check(users, news, 128, rng.choice(keys, MIX_N), 20, S=S)


# ---- 3. m >= k, exclusions, determinism ----
def test_cap_at_or_above_k_is_the_plain_answer_bit_for_bit():
    from newsrec_b200.ops import top_k_scores
    users, news = _mix_inputs(16)
    cat = np.random.default_rng(16).integers(0, 4, MIX_N)
    for k in (1, 10, 100, 128):
        i0, s0 = top_k_scores(users, news, k)
        for m in (k, k + 1, 10 ** 6):
            i1, s1 = _capped(users, news, k, cat, m)
            assert torch.equal(i0, i1) and G._bits_equal(s0, s1), (k, m)
    few_i, few_s = top_k_scores(users[:3], news, 100)                 # several splits: the capped merge kernel
    i1, s1 = _capped(users[:3], news, 100, cat, 100)
    assert torch.equal(few_i, i1) and G._bits_equal(few_s, s1)


def test_exclusions_never_count_against_a_cap():
    users, news = _mix_inputs(17)
    n = MIX_N
    rng = np.random.default_rng(17)
    cat = rng.integers(0, 17, n)
    S = (users.double() @ news.double().T)
    excl = []
    for u in range(MIX_U):
        if u % 3 == 0:
            excl.append([])
        elif u % 3 == 1:                                              # the user's own best 40: they would fill the caps
            excl.append(torch.topk(S[u], 40).indices.numpy()[::-1].copy())
        else:                                                         # every news of the user's best category
            excl.append(np.flatnonzero(cat == cat[int(torch.argmax(S[u]))]))
    S = kernel_scores(users, news)
    for k, m in ((10, 2), (100, 3)):
        _check(users, news, k, cat, m, excl, S=S)
    small = news[:200]
    _check(users[:5], small, 10, cat[:200], 1, [np.arange(200)] * 5)  # everything excluded
    idx, _ = _capped(users[:5], small, 10, cat[:200], 1, [np.arange(200)] * 5)
    assert bool((idx == -1).all())


def test_determinism_and_split_invariance():
    from newsrec_b200.ops import top_k_scores
    g = torch.Generator().manual_seed(18)
    users = torch.randn(9000, 300, generator=g)                      # > 132 user tiles: one split
    news = torch.randn(4097, 300, generator=g)
    cat = np.random.default_rng(18).integers(0, 17, 4097)
    for k, m in ((10, 2), (128, 1)):
        a = _capped(users, news, k, cat, m)
        b = _capped(users, news, k, cat, m)
        assert torch.equal(a[0], b[0]) and G._bits_equal(a[1], b[1])
        for sl in (slice(0, 3), slice(4000, 4005), slice(8990, 9000)):  # few users: several splits and the merge
            few = _capped(users[sl], news, k, cat, m)
            assert torch.equal(few[0], a[0][sl]) and G._bits_equal(few[1], a[1][sl]), (k, m, sl)
    plain = top_k_scores(users[:64], news, 10)
    assert not torch.equal(plain[0], _capped(users[:64], news, 10, cat, 1)[0])  # the cap does bind here


def test_flags_and_refusals_before_any_launch():
    from newsrec_b200 import NewsrecError, launch_count
    from newsrec_b200.ops import top_k_scores
    users, news = torch.randn(4, 30), torch.randn(50, 30)
    cat = torch.zeros(50, dtype=torch.int32)
    n0 = launch_count()
    for m in (0, -1, 2.5, True, None):
        with pytest.raises(NewsrecError):
            top_k_scores(users, news, 10, categories=cat, max_per_category=m)
    with pytest.raises(NewsrecError, match="go together"):
        top_k_scores(users, news, 10, max_per_category=2)
    for bad in (torch.zeros(49, dtype=torch.int32), torch.zeros(50, 1, dtype=torch.int32), torch.zeros(50),
                torch.tensor([2 ** 31] * 50)):
        with pytest.raises(NewsrecError, match="categories|int32"):
            top_k_scores(users, news, 10, categories=bad, max_per_category=2)
    assert launch_count() == n0
    rows, offs = TR._csr([[5], [50], [], []])
    with pytest.raises(IndexError, match="outside the news pool"):
        top_k_scores(users, news, 10, rows, offs, categories=cat, max_per_category=2)
    bad = news.clone()
    bad[7, 3] = float("nan")
    with pytest.raises(ValueError, match="not finite"):
        top_k_scores(users, bad, 10, categories=cat, max_per_category=2)


# ---- 5. the raw entry point ----
def test_guard_bands_of_the_raw_entry_point():
    from newsrec_b200 import launch_count, load_library
    lib = load_library()
    g = torch.Generator().manual_seed(19)
    U, n, D, k, m = 70, 3000, 150, 100, 3
    users = torch.randn(U, D, generator=g).to(DEV)
    news = torch.randn(n, D, generator=g).to(DEV)
    cat = torch.randint(0, 17, (n,), generator=g, dtype=torch.int32).to(DEV)
    ws_bytes = int(lib.nr_topk_dot_workspace(U, n, D, k))
    idx = G._Guarded(U * k, torch.int64, -777, sentinel=-4242)
    score = G._Guarded(U * k, torch.float32, float("nan"))
    ws = G._Guarded(ws_bytes + 256, torch.uint8, 0xAB, sentinel=0x5C)
    flags = G._Guarded(2, torch.int32, 0, sentinel=-3)
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    wp = ws.all.data_ptr()
    pad = (-wp) % 256

    def call(**bad):
        return lib.nr_topk_dot_capped(users.data_ptr(), U, bad.get("ld", D), news.data_ptr(), n, D, bad.get("D", D),
                                      bad.get("k", k), None, None, bad.get("cat", cat.data_ptr()), bad.get("m", m),
                                      idx.all.data_ptr(), score.all.data_ptr(), flags.all.data_ptr(),
                                      flags.all.data_ptr() + 4, wp + pad, bad.get("ws", ws_bytes), s)
    n0 = launch_count()
    assert call() == 0
    torch.cuda.synchronize()
    assert launch_count() > n0
    assert idx.guard_ok() and score.guard_ok() and flags.guard_ok() and ws.guard_ok()
    assert not torch.isnan(score.body).any() and (flags.body == 0).all()
    want_i, want_s = host_walk(kernel_scores(users, news), cat.cpu().numpy(), m, k)
    assert torch.equal(idx.body.view(U, k), want_i) and G._bits_equal(score.body.view(U, k), want_s)
    for bad in [dict(m=0), dict(m=-2), dict(cat=None), dict(k=0), dict(k=129), dict(D=0), dict(ld=D - 1),
                dict(ws=ws_bytes - 1)]:
        before = (idx.body.clone(), score.body.clone())
        n0 = launch_count()
        assert call(**bad) == -1 and lib.nr_last_error().decode().startswith("nr_topk_dot"), bad
        torch.cuda.synchronize()
        assert launch_count() == n0
        assert torch.equal(idx.body, before[0]) and G._bits_equal(score.body, before[1])
        assert idx.guard_ok() and score.guard_ok() and ws.guard_ok()


# ---- 6. end to end ----
@pytest.mark.parametrize("name", ["NRMS", "NAML"])
@pytest.mark.parametrize("field", ["category", "subcategory"])
def test_recommend_diversified(name, field, tmp_path):
    from newsrec_b200 import evaluate as E
    from newsrec_b200.recommend import recommend
    d = str(tmp_path)
    TE._write_validation_dir(d)
    u2i = os.path.join(d, "user2int.tsv")
    model = TR._model(name)
    k, m = 20, 2
    files = {}
    for chunk in (1, 7, 10 ** 9):
        files[chunk] = str(tmp_path / f"rec_{chunk}.tsv")
        n_lines = recommend(model, d, files[chunk], k, user2int_path=u2i, chunk_users=chunk, max_per_category=m,
                            diversify_by=field)
    data = {c: open(f, "rb").read() for c, f in files.items()}
    assert data[1] == data[7] == data[10 ** 9]
    lines = TR._read(files[1])
    assert len(lines) == n_lines
    ids, cols = E.read_news(d, [field])
    key = dict(zip(ids, cols[field].tolist()))
    with torch.no_grad():
        index, matrix = E.news_matrix(model, d)
        beh = E.read_behaviors(d)
        tables = E.build_tables(d, index, model.config.num_clicked_news_a_user, 10 ** 9, u2i)
        uv = E.user_vectors(model, tables, matrix, E.new_flag(matrix.device))
    pad = index["PADDED_NEWS"]
    assert [u for u, _ in lines] == E.distinct_histories(beh)["user"].tolist()
    for _, got in lines:
        _, cnt = np.unique([key[x] for x in got], return_counts=True)
        assert len(got) <= k and (cnt.size == 0 or cnt.max() <= m), got
    elig = torch.ones((len(uv), pad), dtype=torch.bool, device=DEV)
    for u in range(len(uv)):
        h = [int(r) for r in tables.history[u] if r != pad]
        if h:
            elig[u, torch.as_tensor(h, device=DEV)] = False
    want, _ = host_walk(kernel_scores(uv, matrix[:pad]), cols[field], m, k, elig)
    for u, (_, got) in enumerate(lines):
        assert got == [ids[r] for r in want[u].tolist() if r >= 0], u
    # a cap of k or more: the plain file, byte for byte
    plain, big = str(tmp_path / "plain.tsv"), str(tmp_path / "big.tsv")
    recommend(model, d, plain, k, user2int_path=u2i)
    recommend(model, d, big, k, user2int_path=u2i, max_per_category=k, diversify_by=field)
    assert open(plain, "rb").read() == open(big, "rb").read()
