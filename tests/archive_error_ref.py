"""Hi-Fi Ark's archive kernels (csrc/archive.cu) restated stage by stage in fp64, with the fp32 error each value may carry.

The four kernels -- nr_archive_user_fwd / _bwd and nr_archive_score_fwd / _bwd -- are written here once, in the order
archive.cu computes them, over an `Arith` that says how to compute:
- the reference: fp64 values, and next to them the spread of the fp32 error (below);
- an fp32 restatement (torch float32, same stages), and fp64 with TF32- or bf16-rounded product operands: what the
  bound must admit and what it must refuse (tests/test_archive_error_host.py);
- planted mistakes (`plant`): Y without the "+ X" residual, Q normalised over the heads p instead of the history h, the
  scorer's u taken as the mean of the archive rows.

Error model (u = 2^-24, the build's --use_fast_math):
- an n-term fp32 dot product (an fma chain or a tree) adds a rounding error of sd u (sqrt(n) ||a o b||_2 + |a . b|);
- one rounded sum, difference or product adds u |v|;
- __expf adds a relative 2^-22 + u |s - max| (the argument's rounding), the approximate reciprocal and sqrtf 2^-22 each;
- input errors propagate linearly, the softmax Jacobian exactly.

Correlation.  An error in P1, Q or the similarity weights is shared by every column f it multiplies, and the next stage
sums over f again; one row's error reaches every head through the softmax over the history.  Treating such errors as
independent misses the bound by up to sqrt(F).  So the errors are not carried as variances: every rounding site draws
one Rademacher sign per error probe, scaled by its sd, and every stage is evaluated on the clean value (probe 0) and on
`probes` perturbed copies at once.  The perturbations are ~1e-7 relative, so each probe's deviation is the linearised
error, with every correlation the kernels' data flow creates, and sd = the RMS deviation over the probes (an unbiased
estimate of the propagated variance; with 128 probes the worst of 10^5 elements is under-estimated by about 30 % at
most).  The seed is fixed, so a check is reproducible.

A ReLU unit of the scorer whose pre-activation lies within K sd of zero may take either branch: `Ref.slack` holds, per
output element, the sum over such units of what flipping that unit alone changes (the backward is linear in dh once the
forward is fixed, so this bounds every mix of branches).

The bound is |got - ref| <= K sd + slack, elementwise.
"""
from __future__ import annotations

import math

import torch

U = 2.0 ** -24
APPROX = 2.0 ** -22       # __expf, the approximate reciprocal, sqrtf
K = 32                    # the bound in standard deviations
PROBES = 128


def tf32(x):
    """round to TF32's 10-bit mantissa, nearest (ties away, as cvt.rna.tf32.f32)"""
    b = x.float().view(torch.int32)
    return ((b + 0x1000) & ~0x1FFF).view(torch.float32).to(x.dtype)


def bf16(x):
    return x.to(torch.bfloat16).to(x.dtype)


class Arith:
    """How a restatement computes.  dtype: float64 (the reference, rounded operands) or float32 (the fp32 restatement);
    rnd: rounds both operands of every product (None, tf32, bf16); probes: error probes (0: values only).  Computed
    tensors carry a leading probe axis z of size 1 + probes (z = 0 is the clean value); inputs carry none."""

    def __init__(self, dtype=torch.float64, rnd=None, probes=0, seed=1, device="cpu"):
        self.dtype, self.rnd, self.probes, self.device = dtype, rnd, probes, torch.device(device)
        self.Z = 1 + probes
        self.gen = torch.Generator(device=self.device).manual_seed(seed) if probes else None

    def input(self, t):
        return t.to(self.device, self.dtype)

    def err(self, v, sd):
        """v (z, ...) plus, on every probe, one rounding error of size sd with a random sign"""
        if not self.probes:
            return v
        v = v.expand(self.Z, *v.shape[1:])
        sign = torch.randint(0, 2, (self.probes,) + tuple(v.shape[1:]), generator=self.gen, device=self.device).to(self.dtype)
        return torch.cat((v[:1], v[1:] + sd * (2 * sign - 1)), 0)

    def rd(self, v):
        """one rounding of v"""
        return self.err(v, U * v[:1].abs())

    def rel(self, v, r):
        """a relative error of sd r"""
        return self.err(v, r * v[:1].abs())

    def dot(self, eq, a, b, n, more=(), add=None):
        """einsum(eq, a, b) (plus the einsums in `more`, plus add) as one n-term fp32 dot product.  Operands whose
        subscripts start with z carry probes; the result always does.  n broadcasts against the result."""
        r = self.rnd if self.rnd is not None else (lambda t: t)
        v = sq = 0
        for e, x, y in [(eq, a, b)] + list(more):
            lhs, out = e.split("->")
            sx, sy = lhs.split(",")
            if not out.startswith("z"):
                x, sx, out = x.unsqueeze(0), "z" + sx, "z" + out
            e = f"{sx},{sy}->{out}"
            v = v + torch.einsum(e, r(x), r(y))
            if self.probes:
                cx = x[:1] if sx.startswith("z") else x
                cy = y[:1] if sy.startswith("z") else y
                sq = sq + torch.einsum(e, cx * cx, cy * cy)
        if add is not None:
            v = v + add
            if self.probes:
                a0 = add[:1] if add.dim() == v.dim() else add
                sq = sq + a0 * a0
        if not self.probes:
            return v
        n = torch.as_tensor(n, dtype=self.dtype, device=self.device)
        return self.err(v, U * (n.sqrt() * sq.sqrt() + v[:1].abs()))

    def softmax(self, s, dim):
        """as warp_softmax: max subtracted first, __expf, the summed exponentials, the approximate reciprocal, the scaling"""
        d = s - s.amax(dim, keepdim=True)
        e = torch.exp(d)
        if not self.probes:
            return e * (1 / e.sum(dim, keepdim=True))
        e = self.err(e, (APPROX + U * d[:1].abs()) * e[:1])
        t = e.sum(dim, keepdim=True)
        t = self.err(t, U * (math.sqrt(s.shape[dim]) * (e[:1] * e[:1]).sum(dim, keepdim=True).sqrt() + t[:1].abs()))
        return self.rd(e * self.rel(1 / t, APPROX))

    def sd(self, v):
        """the spread of v's error over the probes (zeros without probes)"""
        if not self.probes:
            return torch.zeros_like(v[0])
        return (v[1:] - v[:1]).pow(2).mean(0).sqrt()


class Total:
    """A weight gradient: per-CTA partial rows added by sum_over_seq (eight interleaved warps, a fixed order), here
    accumulated chunk by chunk (per probe, plus the clean rows' squares for the rounding of the final sum)."""

    def __init__(self):
        self.v, self.sq, self.n = 0, 0, 0

    def add(self, part):
        """part (z, rows, ...)"""
        self.v = self.v + part.sum(1)
        self.sq = self.sq + (part[:1] * part[:1]).sum(1)
        self.n += part.shape[1]

    def value(self, ar):
        if not ar.probes:
            return self.v
        return ar.err(self.v, U * (math.sqrt(self.n) * self.sq.sqrt() + self.v[:1].abs()))


# ---- user side: archive_user_fwd_kernel / archive_user_bwd_kernel ------------------------------------------------------------
def user_forward_core(ar, X, W, plant=None):
    """X (b, H, F) input, W (F, P) input -> P1, Y, Q (z, b, ...), as user_forward_core"""
    H, F = X.shape[-2:]
    S = ar.dot("bif,bjf->bij", X, X, F)
    P1 = ar.softmax(S, -1)
    residual = plant != "no_residual"
    Y = ar.dot("zbhi,bif->zbhf", P1, X, H + residual, add=X if residual else None)
    L = ar.dot("zbhf,fp->zbhp", Y, W, F)
    Q = ar.softmax(L, 3 if plant == "q_over_p" else 2)
    return P1, Y, Q


def regularizer(ar, W):
    """G = W^T W and R = ||G * (1 - I)||_F (z, P, P), (z,)"""
    F, P = W.shape
    G = ar.dot("fp,fq->pq", W, W, F)
    Go = G * (1 - torch.eye(P, dtype=ar.dtype, device=ar.device))
    R = torch.sqrt(ar.dot("zpq,zpq->z", Go, Go, max(P * P - P, 1)))
    return G, (ar.rel(R, APPROX) if ar.probes else R)


def user_chunk(ar, X, W, dA=None, reg=None, plant=None):
    """one chunk of users.  X (b, H, F), W (F, P), dA (b, P, F) inputs; reg = (dreg, G, R) when the chunk holds user 0
    (block 0 adds dreg * dR/dW to its partial row).  -> archive, and with dA: dhist and the dW partial rows (z, b, F, P)"""
    H, F = X.shape[-2:]
    P = W.shape[1]
    P1, Y, Q = user_forward_core(ar, X, W, plant)
    out = {"archive": ar.dot("zbhp,zbhf->zbpf", Q, Y, H)}
    if dA is None:
        return out
    dQ = ar.dot("bpf,zbhf->zbhp", dA, Y, F)
    t = ar.dot("zbhp,zbhp->zbp", Q, dQ, H)
    dL = ar.rd(Q * ar.rd(dQ - t.unsqueeze(2)))
    part = ar.dot("zbhf,zbhp->zbfp", Y, dL, H)
    if reg is not None:
        dreg, G, R = reg
        if float(R[0]) > 0 and dreg != 0:
            scale = ar.rel(2 * dreg / R, APPROX) if ar.probes else 2 * dreg / R
            Go = G * (1 - torch.eye(P, dtype=ar.dtype, device=ar.device))
            g = ar.dot("fq,zqp->zfp", W, Go, max(P - 1, 1))
            row0 = ar.rd(part[:, 0] + scale[:, None, None] * g)
            part = torch.cat((row0.unsqueeze(1), part[:, 1:]), 1)
    dY = ar.dot("zbhp,bpf->zbhf", Q, dA, 2 * P, more=[("zbhp,fp->zbhf", dL, W)])
    dP1 = ar.dot("zbif,bjf->zbij", dY, X, F)
    t2 = ar.dot("zbij,zbij->zbi", P1, dP1, H)
    dS = ar.rd(P1 * ar.rd(dP1 - t2.unsqueeze(3)))
    dSs = ar.rd(dS + dS.transpose(2, 3))
    out["dhist"] = ar.dot("zbih,zbif->zbhf", P1, dY, 2 * H + 1, more=[("zbhi,bif->zbhf", dSs, X)], add=dY)
    out["part"] = part
    return out


class Ref:
    """value[name], sd[name] and slack[name] of every output (fp64 or fp32 values, CPU tensors)"""

    def __init__(self):
        self.value, self.sd, self.slack = {}, {}, {}

    def put(self, ar, name, v):
        self.value[name] = v[0].double().cpu()
        self.sd[name] = ar.sd(v).double().cpu()
        self.slack.setdefault(name, torch.zeros_like(self.value[name]))


def _chunks(n, size):
    return [(i, min(i + size, n)) for i in range(0, n, size)]


def user_ref(ar, x, W, darchive=None, dreg=0.0, plant=None, budget=2e7):
    """nr_archive_user_fwd (archive, reg) and, with darchive, nr_archive_user_bwd (dhist, dW).  x (B, H, F), W (F, P),
    darchive (B, P, F), dreg a float."""
    B, H, F = x.shape
    P = W.shape[1]
    Wd = ar.input(W)
    G, R = regularizer(ar, Wd)
    ref, dW = Ref(), Total()
    pieces = {}
    step = max(1, int(budget // (ar.Z * H * (2 * F + 3 * H + 2 * P) + ar.Z * P * F)))
    for lo, hi in _chunks(B, step):
        reg = (dreg, G, R) if lo == 0 else None
        o = user_chunk(ar, ar.input(x[lo:hi]), Wd, None if darchive is None else ar.input(darchive[lo:hi]), reg, plant)
        for k in ("archive", "dhist"):
            if k in o:
                pieces.setdefault(k, []).append((o[k][0], ar.sd(o[k])))
        if "part" in o:
            dW.add(o["part"])
    for k, v in pieces.items():
        ref.value[k] = torch.cat([a for a, _ in v]).double().cpu()
        ref.sd[k] = torch.cat([s for _, s in v]).double().cpu()
        ref.slack[k] = torch.zeros_like(ref.value[k])
    ref.put(ar, "reg", R.reshape(-1, 1))
    if darchive is not None:
        ref.put(ar, "dW", dW.value(ar))
    return ref


# ---- scorer: archive_score_fwd_kernel / archive_score_bwd_kernel --------------------------------------------------------------
def score_chunk(ar, c, owner, A, W1, b1, w2, b2, dlog=None, plant=None, flip=None):
    """The candidates c (n, F) of a run of segments; owner (n,) the segment of each, A (S, P, F) their archives.  -> logits,
    pre (the hidden pre-activations), and with dlog: dcand, darchive and the partial rows pW1, pb1, pw2, pb2 of the
    segments.  flip (n, Hd) bool: take the other ReLU branch at these units."""
    n, F = c.shape
    S, P = A.shape[:2]
    Hd = W1.shape[0]
    Ao = A[owner]
    s = ar.dot("npf,nf->np", Ao, c, F)
    w = ar.softmax(s, 2)
    if plant == "u_mean":
        u = Ao.mean(1).unsqueeze(0).expand(ar.Z, n, F)
    else:
        u = ar.dot("znp,npf->znf", w, Ao, P)
    z = torch.cat((c.unsqueeze(0).expand(ar.Z, n, F), u), 2)
    pre = ar.dot("znj,kj->znk", z, W1, 2 * F + 1, add=b1)
    on = pre[0] > 0
    if flip is not None:
        on = on ^ flip
    h = pre * on
    out = {"logits": ar.dot("znk,k->zn", h, w2, Hd + 1, add=b2), "pre": pre}
    if dlog is None:
        return out
    O = torch.nn.functional.one_hot(owner, S).to(ar.dtype)          # (n, S): exact, a product with it rounds nothing
    cnt = O.sum(0)
    dh = ar.rd((dlog[:, None] * w2).unsqueeze(0)) * on
    out["pb1"] = ar.dot("zik,is->zsk", dh, O, cnt[:, None])
    out["pw2"] = ar.dot("zik,is->zsk", h, O * dlog[:, None], cnt[:, None])
    out["pb2"] = ar.dot("is,i->s", O, dlog, cnt)
    dz = ar.dot("zik,kj->zij", dh, W1, Hd)
    out["pW1"] = ar.dot("zisk,zij->zskj", O[None, :, :, None] * dh[:, :, None, :], z, cnt[:, None, None])
    du = dz[..., F:]
    dw = ar.dot("npf,znf->znp", Ao, du, F)
    t = ar.dot("znp,znp->zn", w, dw, P)
    ds = ar.rd(w * ar.rd(dw - t.unsqueeze(2)))
    out["dcand"] = ar.dot("znp,npf->znf", ds, Ao, P + 1, add=dz[..., :F])
    out["darchive"] = ar.dot("zisp,zif->zspf", O[None, :, :, None] * w[:, :, None, :], du, 2 * cnt[:, None, None],
                             more=[("zisp,if->zspf", O[None, :, :, None] * ds[:, :, None, :], c)])
    return out


WEIGHT_GRADS = ("pW1", "pb1", "pw2", "pb2")


def score_ref(ar, news, seg, archive, W1, b1, w2, b2, dlog=None, plant=None, budget=2e7):
    """nr_archive_score_fwd (logits) and, with dlog, nr_archive_score_bwd (dcand, darchive, dW1, db1, dw2, db2) in the
    NULL-index form: candidate i is news row i.  seg (S + 1,) offsets."""
    F = news.shape[1]
    S, P = archive.shape[:2]
    Hd = W1.shape[0]
    seg = [int(v) for v in seg]
    W1d, b1d, w2d, b2d = (ar.input(t) for t in (W1, b1, w2.reshape(-1), b2.reshape(-1)))
    ref, tot = Ref(), {k: Total() for k in WEIGHT_GRADS}
    pieces = {}
    per_seg = ar.Z * (2 * P * F + 2 * Hd * F)
    per_cand = ar.Z * (P * F // 8 + 4 * F + 4 * Hd) + 3 * P * F
    slack = {}
    s0 = 0
    while s0 < S:                                                   # runs of segments within the budget
        s1 = s0 + 1
        while s1 < S and (s1 + 1 - s0) * per_seg + (seg[s1 + 1] - seg[s0]) * per_cand <= budget:
            s1 += 1
        lo, hi = seg[s0], seg[s1]
        owner = torch.repeat_interleave(torch.arange(s1 - s0), torch.tensor([seg[i + 1] - seg[i] for i in range(s0, s1)]))
        args = (ar.input(news[lo:hi]), owner.to(ar.device), ar.input(archive[s0:s1]), W1d, b1d, w2d, b2d)
        dl = None if dlog is None else ar.input(dlog[lo:hi])
        o = score_chunk(ar, *args, dlog=dl, plant=plant)
        for k in ("logits", "dcand", "darchive"):
            if k in o:
                pieces.setdefault(k, []).append((o[k][0], ar.sd(o[k])))
        for k in WEIGHT_GRADS:
            if k in o:
                tot[k].add(o[k])
        if ar.probes:                                               # ReLU units that may take either branch
            amb = (o["pre"][0].abs() <= K * ar.sd(o["pre"])).nonzero().tolist()
            clean = Arith(ar.dtype, None, 0, device=ar.device)
            for i, k in amb:
                j = int(owner[i])
                a, b = seg[s0 + j] - lo, seg[s0 + j + 1] - lo
                one = (args[0][a:b], torch.zeros(b - a, dtype=torch.long, device=ar.device), args[2][j:j + 1]) + args[3:]
                fl = torch.zeros((b - a, Hd), dtype=torch.bool, device=ar.device)
                fl[i - a, k] = True
                d0 = None if dl is None else dl[a:b]
                x0, x1 = score_chunk(clean, *one, dlog=d0), score_chunk(clean, *one, dlog=d0, flip=fl)
                for name, v in x0.items():
                    if name == "pre":
                        continue
                    dv = (x1[name][0] - v[0]).abs().double().cpu()
                    slack.setdefault(name, []).append((s0 + j, seg[s0 + j], dv))
        s0 = s1
    for k, v in pieces.items():
        ref.value[k] = torch.cat([a for a, _ in v]).double().cpu()
        ref.sd[k] = torch.cat([s for _, s in v]).double().cpu()
        ref.slack[k] = torch.zeros_like(ref.value[k])
    for k in WEIGHT_GRADS:
        if dlog is not None:
            ref.put(ar, "d" + k[1:], tot[k].value(ar).reshape(-1) if k == "pb2" else tot[k].value(ar))
    for name, items in slack.items():
        for s, row0, dv in items:
            if name in ("logits", "dcand"):
                ref.slack[name][row0:row0 + dv.shape[0]] += dv
            elif name == "darchive":
                ref.slack[name][s] += dv[0]
            else:
                key = "d" + name[1:]
                ref.slack[key] += dv[0].reshape(ref.slack[key].shape)
    return ref


def ratios(got, ref, names=None):
    """max over the elements of |got - ref| / (K sd + slack) per output (inf where the bound is 0 and got differs)"""
    res = {}
    for name in names or ref.value:
        g = got[name].double().cpu().reshape(ref.value[name].shape)
        err = (g - ref.value[name]).abs()
        bound = K * ref.sd[name] + ref.slack[name]
        r = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, torch.inf, 0.0))
        r = torch.where(torch.isnan(g), torch.inf, r)
        res[name] = float(r.max()) if r.numel() else 0.0
    return res


def restate(ar, fn, *args, **kw):
    """the outputs of a restatement without probes, as fp64 CPU tensors"""
    r = fn(ar, *args, **kw)
    return {k: v.double() for k, v in r.value.items()}


# ---- the cases both the host test and the kernel test run ---------------------------------------------------------------------
# (H, F, P): F = 400 (every thread of a column loop owns two columns), F % 8 == 4 (row_dot's two accumulators see unequal
# lengths), P > H (the backward stages dA in X's max(H, P) rows), P > 8 warps (the per-head loops wrap), P^2 > 256 threads
# (the regulariser's G loop wraps), P = 1, and the shared-memory corner (50, 400, 32).
USER_CASES = [(1, 8, 5), (6, 8, 5), (50, 8, 5), (1, 300, 5), (6, 300, 5), (50, 300, 5),
              (1, 400, 32), (6, 300, 32), (33, 4, 9), (50, 12, 8), (50, 260, 1), (32, 396, 31), (50, 400, 32)]
# (F, P, hidden): hidden = 1 and 32 (every lane of the w2 . h reduction), the stated corner (400, 32, 32), the shipped
# shape (300, 5, 24), and the earlier int(sqrt(2F)) shapes.
SCORE_CASES = [(8, 5, 4), (300, 5, 24), (300, 1, 24), (400, 32, 28),
               (4, 1, 1), (12, 9, 9), (260, 8, 32), (400, 32, 32)]
SEGMENTS = [5, 1, 13, 0, 300]          # candidates per segment: none, one, 13 and 300


def f32(t):
    """fp64 values that fp32 holds exactly: the kernels' inputs"""
    return t.float().double()


def user_inputs(B, H, F, P, seed=0):
    import newsrec_oracle as O
    x = f32(O.det_uniform((B, H, F), 10 * H + F + seed, -1, 1, torch.float64) * (3.0 / math.sqrt(F)))  # |x| ~ 1.7
    W = f32(O.det_uniform((F, P), 7 + F + P, -0.1, 0.1, torch.float64))
    darchive = f32(O.det_uniform((B, P, F), 900 + seed, -1, 1, torch.float64))
    return x, W, darchive


def score_inputs(F, P, Hd, counts):
    import numpy as np
    import newsrec_oracle as O
    seg = torch.tensor(np.concatenate([[0], np.cumsum(counts)]), dtype=torch.int64)
    S, n = len(counts), int(seg[-1])
    cand = f32(O.det_uniform((n, F), 61 + F, -1, 1, torch.float64) * (3.0 / math.sqrt(F)))
    archive = f32(O.det_uniform((S, P, F), 62 + F, -1, 1, torch.float64) * (3.0 / math.sqrt(F)))
    W1 = f32(O.det_uniform((Hd, 2 * F), 63, -1, 1, torch.float64) / math.sqrt(2 * F))
    b1 = f32(O.det_uniform((Hd,), 64, -0.1, 0.1, torch.float64))
    w2 = f32(O.det_uniform((1, Hd), 65, -1, 1, torch.float64) / math.sqrt(Hd))
    b2 = f32(O.det_uniform((1,), 66, -0.1, 0.1, torch.float64))
    dlog = f32(O.det_uniform((n,), 67, -1, 1, torch.float64))
    return cand, seg, archive, W1, b1, w2, b2, dlog


# the outputs where TF32 or bf16 operands must miss the bound on their own; db1 and db2 sum the incoming gradients, dw2
# averages its rounding over the candidates and the regulariser over P^2 entries, so these four are judged only within
# their kernel's worst element
PRODUCT_OUTPUTS = ("archive", "dhist", "dW", "logits", "dcand", "darchive", "dW1")
