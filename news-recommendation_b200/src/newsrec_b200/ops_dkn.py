"""autograd wrappers, part 4: DKN (csrc/abi_cnn.cu nr_kcnn_encoder_*, csrc/archive.cu nr_dkn_user_*).  Same rules as ops.py:
torch owns memory, streams and autograd bookkeeping; the arithmetic is in the C-ABI kernels.

    KcnnEncoderFn  title word ids + title entity ids (n, T) -> news vectors (n, len(windows) * F)   (reference DKN/KCNN.py)
    DknStepFn      training: news-vector rows -> logits, the gradient of all history and candidate rows in one buffer
    DknUserFn      clicked-news vectors (B, H, F') -> the user vector (B, F')                     (reference DKN/attention.py)
    dkn_score      candidates against user vectors through the archive scorer with a one-row archive
                   (reference general/click_predictor/DNN.py)

Layout: the kernels keep window w of a news vector in columns [w Fs, w Fs + F), Fs = round_up(F, 4), with zero padding
columns (the float4 rows of the pooling backward and of the archive scorer).  Every autograd boundary presents the reference's
compact rows of len(windows) * F columns; _widen / _narrow convert, and the padding columns of every gradient are exact zeros.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import KcnnEncoderBwdArgs, KcnnEncoderFwdArgs, NewsrecError, check, load_library, require_cuda
from .ops import _p, _stream, cast_pad, ru8, ru16, table_operand
from .ops_hifiark import _score_bwd, _score_fwd
from .ops_hifiark import score_impressions as _archive_score_impressions


def _ru4(x: int) -> int:
    return (x + 3) // 4 * 4


def _cols(F: int, n_win: int, device):
    """positions of the compact n_win * F columns in the sectioned n_win * round_up(F, 4) layout"""
    Fs = _ru4(F)
    return (torch.arange(n_win, device=device).view(-1, 1) * Fs + torch.arange(F, device=device).view(1, -1)).reshape(-1)


def _widen(x, F, n_win):
    """(..., n_win * F) -> (..., n_win * Fs) fp32 with zero padding columns (differentiable)"""
    x = x.float()
    out = x.new_zeros(x.shape[:-1] + (n_win * _ru4(F),))
    return out.index_copy(-1, _cols(F, n_win, x.device), x)


def _narrow(x, F, n_win):
    return x.index_select(-1, _cols(F, n_win, x.device))


def _pack_w1(W1, F, n_win):
    """the DNN weight (hidden, 2 n_win F) over [c; u] -> (hidden, 2 n_win Fs), both halves sectioned (differentiable)"""
    Fc = n_win * F
    return torch.cat([_widen(W1[:, :Fc], F, n_win), _widen(W1[:, Fc:], F, n_win)], 1).contiguous()


def _unpack_w1(dW1p, F, n_win):
    Fs = n_win * _ru4(F)
    return torch.cat([_narrow(dW1p[:, :Fs], F, n_win), _narrow(dW1p[:, Fs:], F, n_win)], 1)


class KcnnEncoderFn(torch.autograd.Function):
    """(title, entities) int64 (n, T) -> (n, len(windows) * F): word embedding and tanh(entity embedding M + b) as two channels,
    Conv2d(2, F, (x, d)) per window x (no padding), ReLU, one additive attention shared by the windows, concatenated.
    reference: DKN/KCNN.py:56-117 (use_context=False).  convs: (weight (F, 2, x, d), bias (F,)) of every window, in order."""

    @staticmethod
    def forward(ctx, title, entities, cache, prefix, bad_flag, word_w, entity_w, Mt, mb, Wa, ba, qv, *convs):
        lib = load_library()
        dev = require_cuda()
        n_win = len(convs) // 2
        Ws, bs = convs[0::2], convs[1::2]
        Fn, chans, _, d = Ws[0].shape
        wins = [int(W.shape[2]) for W in Ws]
        if chans != 2:
            raise NewsrecError(f"KCNN: {chans} input channels; the kernels implement word + entity (use_context=False)")
        de, q = Mt.shape[0], Wa.shape[0]
        sec, lde, ldf, ldq, Fs = ru8(d + 1), ru8(de + 1), ru8(Fn + 1), ru16(q), _ru4(Fn)
        ldx, Kt, taps = 2 * sec, n_win * ldf, max(wins)
        n_seq, T = title.shape

        def build(Mt, mb, Wa, ba, qv, *convs):
            Ws, bs = convs[0::2], convs[1::2]
            wconv = torch.zeros((sum(wins) * Fn, ldx), dtype=torch.float32, device=dev)
            wT = torch.zeros((2, taps, d, Kt), dtype=torch.float32, device=dev)
            r = 0
            for w, W in enumerate(Ws):
                for s in range(wins[w]):
                    wconv[r:r + Fn, :d] = W[:, 0, s]
                    wconv[r:r + Fn, sec:sec + d] = W[:, 1, s]
                    r += Fn
                    for c in range(2):  # tap taps - 1 - s of the transposed conv reads dY[row - s]
                        wT[c, taps - 1 - s, :, w * ldf:w * ldf + Fn] = W[:, c, s].t()
            return dict(wconv=cast_pad(wconv, ldx), bconv=torch.cat([b.float() for b in bs]).contiguous(),
                        wT_word=cast_pad(wT[0].reshape(taps * d, Kt), Kt), wT_entity=cast_pad(wT[1].reshape(taps * d, Kt), Kt),
                        mT=cast_pad(Mt, lde, transpose=True), m=cast_pad(Mt, sec), mb=mb.float().contiguous(),
                        wa=cast_pad(Wa, ldf), waT=cast_pad(Wa, ldq, transpose=True), ba=ba.float().contiguous(),
                        qv=qv.float().contiguous())

        ops = cache.get(prefix, (Mt, mb, Wa, ba, qv) + tuple(convs), build)
        word_t = table_operand(cache, prefix + ".word", word_w)
        ent_t = table_operand(cache, prefix + ".entity", entity_w)
        title, entities = title.contiguous(), entities.contiguous()
        rows = n_seq * sum(T + 1 - x for x in wins)
        X2 = torch.empty((n_seq * T, ldx), dtype=torch.bfloat16, device=dev)
        E = torch.empty((n_seq * T, lde), dtype=torch.bfloat16, device=dev)
        Y = torch.empty((rows, ldf), dtype=torch.bfloat16, device=dev)
        w = torch.empty((rows,), dtype=torch.float32, device=dev)
        out = torch.empty((n_seq, n_win * Fs), dtype=torch.float32, device=dev)
        a = KcnnEncoderFwdArgs()
        a.n_seq, a.T, a.d, a.de, a.F, a.q, a.n_win = n_seq, T, d, de, Fn, q, n_win
        a.win = (C.c_int * 4)(*(wins + [0] * (4 - n_win)))
        a.ldx, a.lde, a.ldf, a.ldo = ldx, lde, ldf, n_win * Fs
        a.word_ids, a.entity_ids, a.word_table_bf16, a.V = _p(title), _p(entities), _p(word_t), word_w.shape[0]
        a.entity_table_bf16, a.Ve = _p(ent_t), entity_w.shape[0]
        a.mT_bf16, a.mb, a.wconv_bf16, a.bconv = _p(ops["mT"]), _p(ops["mb"]), _p(ops["wconv"]), _p(ops["bconv"])
        a.wa_bf16, a.ba, a.qv = _p(ops["wa"]), _p(ops["ba"]), _p(ops["qv"])
        a.X2_bf16, a.E_bf16, a.Y_bf16, a.w, a.out, a.bad_id_flag = _p(X2), _p(E), _p(Y), _p(w), _p(out), _p(bad_flag)
        check(lib.nr_kcnn_encoder_fwd(C.byref(a), _stream()), "nr_kcnn_encoder_fwd")
        ctx.save_for_backward(title, entities, X2, E, Y, w)
        ctx.meta = dict(n_seq=n_seq, T=T, d=d, de=de, F=Fn, q=q, wins=wins, ops=ops, V=word_w.shape[0], Ve=entity_w.shape[0])
        return _narrow(out, Fn, n_win)

    @staticmethod
    def backward(ctx, dout):
        lib = load_library()
        title, entities, X2, E, Y, w = ctx.saved_tensors
        m = ctx.meta
        dev = X2.device
        n_seq, T, d, de, Fn, q, wins, ops = m["n_seq"], m["T"], m["d"], m["de"], m["F"], m["q"], m["wins"], m["ops"]
        n_win = len(wins)
        sec, lde, ldf, ldq = ru8(d + 1), ru8(de + 1), ru8(Fn + 1), ru16(q)
        ldx = 2 * sec
        g = _widen(dout.contiguous(), Fn, n_win)
        dWc = torch.zeros((sum(wins) * Fn, ldx), dtype=torch.float32, device=dev)
        dM = torch.zeros((d, lde), dtype=torch.float32, device=dev)
        dWa = torch.zeros((q, ldf), dtype=torch.float32, device=dev)
        dqv = torch.zeros((q,), dtype=torch.float32, device=dev)
        dword = torch.zeros((m["V"], d), dtype=torch.float32, device=dev)
        dent = torch.zeros((m["Ve"], de), dtype=torch.float32, device=dev)
        ws_bytes = int(lib.nr_kcnn_encoder_bwd_workspace(n_seq, T, d, Fn, q, n_win))
        ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
        a = KcnnEncoderBwdArgs()
        a.n_seq, a.T, a.d, a.de, a.F, a.q, a.n_win = n_seq, T, d, de, Fn, q, n_win
        a.win = (C.c_int * 4)(*(wins + [0] * (4 - n_win)))
        a.ldx, a.lde, a.ldf, a.ldo, a.ldq = ldx, lde, ldf, g.shape[1], ldq
        a.word_ids, a.entity_ids, a.V, a.Ve = _p(title), _p(entities), m["V"], m["Ve"]
        a.wT_word_bf16, a.wT_entity_bf16, a.m_bf16 = _p(ops["wT_word"]), _p(ops["wT_entity"]), _p(ops["m"])
        a.wa_bf16, a.waT_bf16, a.ba, a.qv = _p(ops["wa"]), _p(ops["waT"]), _p(ops["ba"]), _p(ops["qv"])
        a.X2_bf16, a.E_bf16, a.Y_bf16, a.w, a.dout = _p(X2), _p(E), _p(Y), _p(w), _p(g)
        a.dWconv_ext, a.dM_ext, a.dWa_ext, a.dqv, a.dword, a.dentity = _p(dWc), _p(dM), _p(dWa), _p(dqv), _p(dword), _p(dent)
        a.workspace, a.workspace_bytes = _p(ws), ws_bytes
        check(lib.nr_kcnn_encoder_bwd(C.byref(a), _stream()), "nr_kcnn_encoder_bwd")
        dconvs, r = [], 0
        for x in wins:
            blk = dWc[r * Fn:(r + x) * Fn].view(x, Fn, ldx)
            dconvs.append(torch.stack([blk[:, :, :d], blk[:, :, sec:sec + d]], 0).permute(2, 0, 1, 3).contiguous())  # (F, 2, x, d)
            dconvs.append(blk[0, :, sec + d].contiguous())
            r += x
        return (None, None, None, None, None, dword, dent, dM[:, :de].t().contiguous(), dM[:, de].contiguous(),
                dWa[:, :Fn].contiguous(), dWa[:, Fn].contiguous(), dqv) + tuple(dconvs)


def _user_fwd(x, W1, w2):
    """x (B, H, F) fp32 contiguous, W1 (hidden, 2F) fp32, w2 (hidden,) -> user (B, F)"""
    lib = load_library()
    B, H, Fn = x.shape
    if W1.shape[1] != 2 * Fn:
        raise NewsrecError(f"DKN attention weight of shape {tuple(W1.shape)} for news vectors of width {Fn}")
    user = torch.empty((B, Fn), dtype=torch.float32, device=x.device)
    check(lib.nr_dkn_user_fwd(_p(x), B, H, Fn, _p(W1), W1.shape[0], _p(w2), _p(user), _stream()), "nr_dkn_user_fwd")
    return user


def _user_bwd(x, W1, w2, duser, dhist):
    """dhist (=, any (B*H, F) row block of fp32 storage); returns (dW1 (hidden, 2F) with exact zeros in the candidate half, dw2)"""
    lib = load_library()
    B, H, Fn = x.shape
    dW1 = torch.zeros_like(W1)
    dw2 = torch.zeros_like(w2)
    ws_bytes = int(lib.nr_dkn_user_bwd_workspace(B, Fn))
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=x.device)
    check(lib.nr_dkn_user_bwd(_p(x), B, H, Fn, _p(W1), W1.shape[0], _p(w2), _p(duser), _p(dhist), _p(dW1), _p(dw2), _p(ws), ws_bytes,
                              _stream()), "nr_dkn_user_bwd")
    return dW1, dw2


def _f32(t):
    return t.detach().float().contiguous()


class DknStepFn(torch.autograd.Function):
    """The training step after the news encoder.  vec (B*H + B*C, n_win*F): the B*H history rows, then the B*C candidate rows
    -> logits (B, C).  The history attention (W1a (16, 2 n_win F), b1a, w2a (1, 16), b2a) gives one user vector per user; the
    DNN click predictor (W1, b1, w2, b2) scores [c; u] through the archive scorer with a one-row archive.  The backward writes
    the gradient of every row of vec into ONE buffer; the gradients of W1a[:, :n_win F], b1a and b2a are exact zeros."""

    @staticmethod
    def forward(ctx, vec, B, H, C, F, n_win, W1a, b1a, w2a, b2a, W1, b1, w2, b2):
        require_cuda()
        v = _widen(vec.detach(), F, n_win).contiguous()
        Fs = v.shape[1]
        W1a_p, w2a_f = _f32(_pack_w1(W1a.detach(), F, n_win)), _f32(w2a).view(-1)
        ops = (_f32(_pack_w1(W1.detach(), F, n_win)), _f32(b1), _f32(w2).view(-1), _f32(b2))
        user = _user_fwd(v[:B * H].view(B, H, Fs), W1a_p, w2a_f)
        seg = torch.arange(0, B * C + 1, C, dtype=torch.int64, device=v.device)
        archive = user.view(B, 1, Fs)
        logits = _score_fwd(v[B * H:], seg, archive, ops)
        ctx.save_for_backward(v, W1a_p, w2a_f, seg, archive, *ops)
        ctx.meta = (B, H, F, n_win)
        return logits.view(B, C)

    @staticmethod
    def backward(ctx, dlogits):
        v, W1a_p, w2a_f, seg, archive, *ops = ctx.saved_tensors
        B, H, F, n_win = ctx.meta
        Fs = v.shape[1]
        dvec = torch.empty_like(v)
        # the packed operands have no gradient storage of their own: the scorer adds into fresh buffers it returns
        darchive, (dW1, db1, dw2, db2) = _score_bwd(v[B * H:], seg, archive, ops, ops, dlogits.reshape(-1).float().contiguous(),
                                                    dvec[B * H:])
        dW1a_p, dw2a = _user_bwd(v[:B * H].view(B, H, Fs), W1a_p, w2a_f, darchive.view(B, Fs).contiguous(), dvec[:B * H])
        zero = torch.zeros(1, dtype=torch.float32, device=v.device)
        return (_narrow(dvec, F, n_win), None, None, None, None, None, _unpack_w1(dW1a_p, F, n_win), zero.expand(dW1a_p.shape[0]).clone(),
                dw2a.view(1, -1), zero.clone(), _unpack_w1(dW1, F, n_win), db1, dw2.view(1, -1), db2)


class DknUserFn(torch.autograd.Function):
    """hist (B, H, F'), any strides; W1a (16, 2F'), w2a (1, 16) -> user (B, F') = sum_j softmax_j(beta . h_j) h_j.
    reference DKN/attention.py, which gives this same vector for every candidate (include/newsrec_b200.h)."""

    @staticmethod
    def forward(ctx, hist, W1a, w2a):
        require_cuda()
        x, W1, w2 = hist.float().contiguous(), _f32(W1a), _f32(w2a).view(-1)
        user = _user_fwd(x, W1, w2)
        ctx.save_for_backward(x, W1, w2)
        return user

    @staticmethod
    def backward(ctx, duser):
        x, W1, w2 = ctx.saved_tensors
        dhist = torch.empty_like(x)
        dW1, dw2 = _user_bwd(x, W1, w2, duser.float().contiguous(), dhist)
        return dhist, dW1, dw2.view(1, -1)


def dkn_score(cand, user, F, n_win, W1, b1, w2, b2):
    """cand (n, n_win F) against one user vector (n_win F,) -> logits (n,): the DNN predictor on [c; u] (differentiable)."""
    from .ops_hifiark import ArchiveScoreFn
    seg = torch.tensor([0, cand.shape[0]], dtype=torch.int64, device=cand.device)
    return ArchiveScoreFn.apply(_widen(cand, F, n_win), seg, _widen(user, F, n_win).view(1, 1, -1), _pack_w1(W1, F, n_win), b1, w2, b2)


def score_impressions(news_matrix, cand_index, seg_offsets, hist, F, n_win, W1a, w2a, W1, b1, w2, b2, bad_flag):
    """Evaluation: every impression in one launch per stage.  hist (S, H, n_win F) the history rows of each impression's user
    -> user vectors (S, n_win F) -> the scores (n_cand,) of the candidates news_matrix[cand_index] (see ops_hifiark)."""
    dev = require_cuda()
    users = _user_fwd(hist.to(dev).float().contiguous(), _f32(W1a), _f32(w2a).view(-1))
    news = _widen(news_matrix.to(dev), F, n_win).contiguous()
    archives = _widen(users, F, n_win).unsqueeze(1).contiguous()
    return _archive_score_impressions(news, cand_index, seg_offsets, archives, _pack_w1(W1.detach(), F, n_win), b1, w2, b2, bad_flag)
