"""autograd wrappers, part 3: Hi-Fi Ark after the news encoder (csrc/archive.cu).  Same rules as ops.py: torch owns memory,
streams and autograd bookkeeping; the arithmetic is in the C-ABI kernels.

    ArchiveStepFn   training: news-vector rows -> logits and the OMAP regulariser, the gradient of all rows in one buffer
    ArchiveUserFn   clicked-news vectors (B, H, F) -> archive (B, P, F)
                    (reference general/attention/self.py + HiFiArk/OMAP.py)
    ArchiveScoreFn  candidate rows against the archive of their segment -> logits
                    (reference general/attention/similarity.py + general/click_predictor/DNN.py)
"""
from __future__ import annotations

import torch

from . import NewsrecError, check, load_library, require_cuda
from .ops import _p, _stream, grad_sink


def _grad_dst(p):
    """(buffer the kernels add the gradient of p into, whether it is p's own storage) -- the grad_sink convention."""
    g = grad_sink(p)
    if g is not None:
        return g, True
    return torch.zeros(p.shape, dtype=torch.float32, device=p.device), False


def _f32(t):
    return t.detach().float().contiguous()


def _user_fwd(x, Wf, with_reg):
    """x (B, H, F) fp32 contiguous, Wf (F, P) -> (archive (B, P, F), regulariser 0-dim; left 0 when with_reg is False)."""
    lib = load_library()
    B, H, Fn = x.shape
    if Wf.shape[0] != Fn:
        raise NewsrecError(f"OMAP weight of shape {tuple(Wf.shape)} for news vectors of width {Fn}")
    P = Wf.shape[1]
    archive = torch.empty((B, P, Fn), dtype=torch.float32, device=x.device)
    reg = torch.zeros((), dtype=torch.float32, device=x.device)
    check(lib.nr_archive_user_fwd(_p(x), B, H, Fn, P, _p(Wf), _p(archive), _p(reg) if with_reg else None, _stream()),
          "nr_archive_user_fwd")
    return archive, reg


def _user_bwd(x, Wf, W, darchive, dreg, dhist):
    """dhist (=, any (B*H, F) row block of fp32 storage); returns W's gradient, or None if it went into W's own .grad."""
    lib = load_library()
    B, H, Fn = x.shape
    P = Wf.shape[1]
    dW, direct = _grad_dst(W)
    ws_bytes = int(lib.nr_archive_user_bwd_workspace(B, Fn, P))
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=x.device)
    check(lib.nr_archive_user_bwd(_p(x), B, H, Fn, P, _p(Wf), _p(darchive), _p(dreg), _p(dhist), _p(dW), _p(ws), ws_bytes,
                                  _stream()), "nr_archive_user_bwd")
    return None if direct else dW


def _dnn_operands(W1, b1, w2, b2):
    return (_f32(W1), _f32(b1), _f32(w2).view(-1), _f32(b2))


def _score_fwd(c, seg, a, ops):
    lib = load_library()
    n, Fn = c.shape
    S, P, Fa = a.shape
    if Fa != Fn or ops[0].shape[1] != 2 * Fn or seg.numel() != S + 1:
        raise NewsrecError(f"archive scorer: candidates {tuple(c.shape)}, archive {tuple(a.shape)}, W1 {tuple(ops[0].shape)}, "
                           f"{seg.numel()} segment offsets")
    logits = torch.empty((n,), dtype=torch.float32, device=c.device)
    check(lib.nr_archive_score_fwd(_p(c), n, Fn, None, n, _p(seg), S, _p(a), P, _p(ops[0]), _p(ops[1]), ops[0].shape[0], _p(ops[2]),
                                   _p(ops[3]), _p(logits), None, _stream()), "nr_archive_score_fwd")
    return logits


def _score_bwd(c, seg, a, ops, params, dlogits, dcand):
    """dcand (=, any (n, F) row block of fp32 storage); returns (darchive, gradients of params or None where they went into
    the parameters' own .grad)."""
    lib = load_library()
    n, Fn = c.shape
    S, P, _ = a.shape
    Hd = ops[0].shape[0]
    darchive = torch.empty_like(a)
    dsts = [_grad_dst(p) for p in params]
    ws_bytes = int(lib.nr_archive_score_bwd_workspace(S, Fn, Hd))
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=c.device)
    check(lib.nr_archive_score_bwd(_p(c), n, Fn, None, n, _p(seg), S, _p(a), P, _p(ops[0]), _p(ops[1]), Hd, _p(ops[2]), _p(ops[3]),
                                   _p(dlogits.float().contiguous()), _p(dcand), _p(darchive), *[_p(d) for d, _ in dsts], _p(ws),
                                   ws_bytes, _stream()), "nr_archive_score_bwd")
    return darchive, tuple(None if direct else d for d, direct in dsts)


class ArchiveStepFn(torch.autograd.Function):
    """The training step after the news encoder.  vec (B*H + B*C, F): the B*H history rows, then the B*C candidate rows (the
    order the batch is packed in) -> (logits (B, C), regulariser 0-dim).  The backward writes the gradient of every row of vec
    into ONE buffer: the scorer its candidate rows, the user side its history rows."""

    @staticmethod
    def forward(ctx, vec, B, H, C, W, W1, b1, w2, b2, with_reg):
        require_cuda()
        v = vec.float().contiguous()
        Fn = v.shape[1]
        Wf, ops = _f32(W), _dnn_operands(W1, b1, w2, b2)
        x, cand = v[:B * H].view(B, H, Fn), v[B * H:]
        archive, reg = _user_fwd(x, Wf, with_reg)
        seg = torch.arange(0, B * C + 1, C, dtype=torch.int64, device=v.device)
        logits = _score_fwd(cand, seg, archive, ops)
        ctx.save_for_backward(v, Wf, seg, archive, *ops)
        ctx.meta = (B, H, bool(with_reg), W, (W1, b1, w2, b2))
        if not with_reg:
            ctx.mark_non_differentiable(reg)
        return logits.view(B, C), reg

    @staticmethod
    def backward(ctx, dlogits, dreg):
        v, Wf, seg, archive, *ops = ctx.saved_tensors
        B, H, with_reg, W, params = ctx.meta
        dvec = torch.empty_like(v)
        darchive, dparams = _score_bwd(v[B * H:], seg, archive, ops, params, dlogits.reshape(-1), dvec[B * H:])
        dreg = dreg.float().contiguous() if (with_reg and dreg is not None) else None
        dW = _user_bwd(v[:B * H].view(B, H, -1), Wf, W, darchive, dreg, dvec[:B * H])
        return (dvec, None, None, None, dW) + dparams + (None,)


class ArchiveUserFn(torch.autograd.Function):
    """get_user_vector: hist (B, H, F), any strides, W (F, P) -> archive (B, P, F)."""

    @staticmethod
    def forward(ctx, hist, W):
        require_cuda()
        x, Wf = hist.float().contiguous(), _f32(W)
        archive, _ = _user_fwd(x, Wf, False)
        ctx.save_for_backward(x, Wf)
        ctx.W = W
        return archive

    @staticmethod
    def backward(ctx, darchive):
        x, Wf = ctx.saved_tensors
        dhist = torch.empty_like(x)
        dW = _user_bwd(x, Wf, ctx.W, darchive.float().contiguous(), None, dhist)
        return dhist, dW


class ArchiveScoreFn(torch.autograd.Function):
    """get_prediction: cand (n, F) candidate rows, seg_offsets (S + 1,) int64 on the device, archive (S, P, F), DNN parameters
    W1 (hidden, 2F), b1 (hidden,), w2 (1, hidden), b2 (1,) -> logits (n,); rows seg_offsets[s] .. seg_offsets[s+1] are scored
    against archive[s]."""

    @staticmethod
    def forward(ctx, cand, seg_offsets, archive, W1, b1, w2, b2):
        require_cuda()
        c, a, ops = cand.float().contiguous(), archive.float().contiguous(), _dnn_operands(W1, b1, w2, b2)
        logits = _score_fwd(c, seg_offsets, a, ops)
        ctx.save_for_backward(c, seg_offsets, a, *ops)
        ctx.params = (W1, b1, w2, b2)
        return logits

    @staticmethod
    def backward(ctx, dlogits):
        c, seg, a, *ops = ctx.saved_tensors
        dcand = torch.empty_like(c)
        darchive, dparams = _score_bwd(c, seg, a, ops, ctx.params, dlogits, dcand)
        return (dcand, None, darchive) + dparams


def score_impressions(news_matrix, cand_index, seg_offsets, archives, W1, b1, w2, b2, bad_flag):
    """Evaluation: scores of many impressions in one launch.  news_matrix (n_news, F), cand_index (n_cand,) int64 rows of the
    candidates of all impressions back to back, seg_offsets (S + 1,), archives (S, P, F) the archive of each impression's user.
    Returns (n_cand,) fp32; a candidate row outside the news matrix sets the device int bad_flag (checked by the caller)."""
    lib = load_library()
    dev = require_cuda()
    news = news_matrix.to(dev).float().contiguous()
    a = archives.to(dev).float().contiguous()
    cand = cand_index.to(dev).long().contiguous()
    seg = seg_offsets.to(dev).long().contiguous()
    S, P, Fn = a.shape
    if seg.numel() != S + 1 or news.shape[1] != Fn:
        raise NewsrecError("score_impressions: archives must be (len(seg_offsets) - 1, P, F) with the news matrix's F")
    ops = _dnn_operands(W1, b1, w2, b2)
    scores = torch.empty((cand.numel(),), dtype=torch.float32, device=dev)
    check(lib.nr_archive_score_fwd(_p(news), news.shape[0], Fn, _p(cand), cand.numel(), _p(seg), S, _p(a), P, _p(ops[0]), _p(ops[1]),
                                   ops[0].shape[0], _p(ops[2]), _p(ops[3]), _p(scores), _p(bad_flag), _stream()), "nr_archive_score_fwd")
    return scores
