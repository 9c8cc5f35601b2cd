"""fp64 restatement of the archive DNN click score over a whole pool (nr_topk_archive, nr_pool_ranks_archive) and of the
per-pair bound include/newsrec_b200.h states for it, shared by the GPU tests of both kernels.

    w = softmax_p(A_u[p] . c)   (P = 1: w = 1),   score = b2 + sum_j w2_j relu(X_j + sum_p w_p Y_pj),
    X = W1[:, :F] c + b1,   Y_p = W1[:, F:] A_u[p]
"""
import torch

U_RND = 2.0 ** -24


def gamma(n):
    return n * U_RND / (1 - n * U_RND)


def operands(g, U, P, F, hidden, n, scale=1.0):
    """Seeded fp32 operands at the scale of trained models: (archive (U, P, F), news (n, F), (W1, b1, w2, b2))."""
    A = torch.randn(U, P, F, generator=g) * scale
    C = torch.randn(n, F, generator=g) * scale
    W1 = torch.randn(hidden, 2 * F, generator=g) / (2 * F) ** 0.5
    b1 = torch.randn(hidden, generator=g) * 0.1
    w2 = torch.randn(1, hidden, generator=g) / hidden ** 0.5
    b2 = torch.randn(1, generator=g) * 0.1
    return A, C, (W1, b1, w2, b2)


def exact_and_bound(A, C, dnn, device, chunk_bytes=1 << 29):
    """(S, E) fp64 (U, n) on device: the exact score of the fp32 inputs and the kernel's stated bound e per pair."""
    W1, b1, w2, b2 = (t.detach().to(device).double() for t in dnn)
    A, C = A.to(device).double(), C.to(device).double()
    U, P, F = A.shape
    n, hid = C.shape[0], W1.shape[0]
    W1c, W1u, b1, w2, b2 = W1[:, :F], W1[:, F:], b1.reshape(-1), w2.reshape(-1), b2.reshape(-1)
    coef = 2.0 ** -15 + 3 * ((F + 63) // 64 * 64) * 2.0 ** -23
    X = C @ W1c.T + b1
    dX = gamma(F + 1) * (C.abs() @ W1c.abs().T + b1.abs())
    S = torch.empty(U, n, dtype=torch.float64, device=device)
    E = torch.empty_like(S)
    uc = max(1, chunk_bytes // max(1, n * max(P, hid) * 8 * 4))
    for a in range(0, U, uc):
        Ac = A[a:a + uc]
        Y = Ac @ W1u.T                                            # (u, P, hid)
        dY = gamma(F) * (Ac.abs() @ W1u.abs().T)
        Ya = Y.abs() + dY
        if P == 1:
            W = torch.ones(Ac.shape[0], n, 1, dtype=torch.float64, device=device)
            ew = torch.zeros(Ac.shape[0], n, dtype=torch.float64, device=device)
        else:
            L = torch.einsum("upf,nf->unp", Ac, C)
            d = coef * torch.einsum("upf,nf->unp", Ac.abs(), C.abs())
            W = torch.softmax(L, -1)
            dmax = d.amax(-1)
            Lmax = L.amax(-1, keepdim=True)
            ew = (1 + 2.0 ** -10) * (2 * dmax + 2 * (W * (2 + 2 * (L - Lmax).abs() + 4 * dmax[..., None])).sum(-1) * 2.0 ** -23
                                     + gamma(P + 2))
        PRE = X[None] + torch.einsum("unp,uph->unh", W, Y)
        Ej = (dX[None] + torch.einsum("unp,uph->unh", W, dY) + ew[..., None] * Ya.amax(1)[:, None, :]
              + gamma(P) * (X.abs()[None] + dX[None] + torch.einsum("unp,uph->unh", W + ew[..., None], Ya)))
        S[a:a + uc] = PRE.clamp(min=0) @ w2 + b2
        E[a:a + uc] = Ej @ w2.abs() + gamma(hid) * (b2.abs() + (PRE.abs() + Ej) @ w2.abs())
    return S, E


def capped_walk(scores, rows, cats, k, m):
    """The host capped walk over one user's (score, row) pairs already in output order: take a row iff fewer than m taken
    share its category and fewer than k are taken."""
    taken, per = [], {}
    for s, r in zip(scores, rows):
        if len(taken) == k:
            break
        c = int(cats[r])
        if per.get(c, 0) < m:
            per[c] = per.get(c, 0) + 1
            taken.append((s, r))
    return taken
