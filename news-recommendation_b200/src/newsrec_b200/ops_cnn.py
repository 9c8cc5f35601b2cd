"""autograd wrappers, part 2: the CNN text encoder (NAML / LSTUR / TANR), generic Linear over dense rows,
fp32 embedding lookups and NAML's category "element" encoder.  Same rules as ops.py: torch owns memory,
streams and autograd bookkeeping; the arithmetic is in the C-ABI kernels."""
from __future__ import annotations

import ctypes as C

import torch

from . import CnnEncoderBwdArgs, CnnEncoderFwdArgs, check, load_library, require_cuda
from .ops import _p, _stream, cast_pad, next_seed, ru8, ru16, table_operand


class CnnPoolEncoderFn(torch.autograd.Function):
    """ids (n_seq, T) int64 -> (n_seq, F):  embedding -> dropout -> Conv2d(1,F,(w,d), padding ((w-1)/2, 0)) -> ReLU -> dropout
    -> additive pool, w = 1 .. 4 from the weight's shape; the pool runs over the L = T + 2 ((w-1)/2) - w + 1 conv outputs.
    reference: NAML/news_encoder.py:21-37, LSTUR/news_encoder.py:56-72, TANR/news_encoder.py:40-52."""

    @staticmethod
    def forward(ctx, ids, emb_w, Wc, bc, Wa, ba, qv, p_drop, cache, prefix, bad_flag, accurate=False):
        lib = load_library()
        dev = require_cuda()
        Fn, _, win, d = Wc.shape  # the C ABI refuses a window outside 1 .. 4 (make_title_cnn already has)
        q = Wa.shape[0]
        ldx, ldf, ldq = ru8(d + 1), ru8(Fn + 1), ru16(q)
        n_seq, T = ids.shape
        L = T + 2 * ((win - 1) // 2) - win + 1
        ids = ids.contiguous()

        def build(Wc, bc, Wa, ba, qv):
            taps = Wc[:, 0]                                                           # (F, w, d)
            wconv = taps.permute(1, 0, 2).reshape(win * Fn, d)                        # tap-major rows
            wconvT = torch.cat([taps[:, win - 1 - s, :].t() for s in range(win)], 0)  # (w d, F): tap s' = W_(w-1-s')^T
            return dict(wconv=cast_pad(wconv, ldx), wconvT=cast_pad(wconvT, ldf), bconv=bc.float().contiguous(),
                        wa=cast_pad(Wa, ldf), waT=cast_pad(Wa, ldq, transpose=True), ba=ba.float().contiguous(),
                        qv=qv.float().contiguous())

        ops = cache.get(prefix, (Wc, bc, Wa, ba, qv), build)
        table = table_operand(cache, prefix + ".table", emb_w)
        Xp = torch.empty((n_seq * (T + 2), ldx), dtype=torch.bfloat16, device=dev)
        Y = torch.empty((n_seq * L, ldf), dtype=torch.bfloat16, device=dev)
        w = torch.empty((n_seq * L,), dtype=torch.float32, device=dev)
        out = torch.empty((n_seq, Fn), dtype=torch.float32, device=dev)
        seed = next_seed() if p_drop > 0 else 0
        a = CnnEncoderFwdArgs()
        a.n_seq, a.T, a.d, a.F, a.q, a.ldx, a.ldf, a.window = n_seq, T, d, Fn, q, ldx, ldf, win
        a.ids, a.table_bf16, a.V = _p(ids), _p(table), emb_w.shape[0]
        a.wconv_bf16, a.bconv, a.wa_bf16, a.ba, a.qv = _p(ops["wconv"]), _p(ops["bconv"]), _p(ops["wa"]), _p(ops["ba"]), _p(ops["qv"])
        a.p_drop, a.seed = float(p_drop), seed
        a.Xp_bf16, a.Y_bf16, a.w, a.out, a.bad_id_flag = _p(Xp), _p(Y), _p(w), _p(out), _p(bad_flag)
        Y_lo = None
        if accurate:  # the conv output as a hi/lo bf16 pair: the pooled sum reads both planes (DESIGN.md section 4)
            Y_lo = torch.empty((n_seq * L, ldf), dtype=torch.bfloat16, device=dev)
            a.Y_lo_bf16 = _p(Y_lo)
        check(lib.nr_cnn_encoder_fwd(C.byref(a), _stream()), "nr_cnn_encoder_fwd")
        ctx.save_for_backward(Xp, Y, w, ids)
        ctx.meta = dict(n_seq=n_seq, T=T, d=d, F=Fn, q=q, win=win, p_drop=float(p_drop), seed=seed, ops=ops, V=emb_w.shape[0])
        return out

    @staticmethod
    def backward(ctx, dout):
        lib = load_library()
        Xp, Y, w, ids = ctx.saved_tensors
        m = ctx.meta
        dev = Xp.device
        n_seq, T, d, Fn, q, win, ops = m["n_seq"], m["T"], m["d"], m["F"], m["q"], m["win"], m["ops"]
        ldx, ldf, ldq = ru8(d + 1), ru8(Fn + 1), ru16(q)
        dout = dout.contiguous().float()
        dWc = torch.zeros((win, Fn, ldx), dtype=torch.float32, device=dev)
        dWa = torch.zeros((q, ldf), dtype=torch.float32, device=dev)
        dqv = torch.zeros((q,), dtype=torch.float32, device=dev)
        demb = torch.zeros((m["V"], d), dtype=torch.float32, device=dev)
        ws_bytes = int(lib.nr_cnn_encoder_bwd_workspace(n_seq, T, Fn, q))
        ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
        a = CnnEncoderBwdArgs()
        a.n_seq, a.T, a.d, a.F, a.q, a.ldx, a.ldf, a.ldq, a.window = n_seq, T, d, Fn, q, ldx, ldf, ldq, win
        a.ids, a.V = _p(ids), m["V"]
        a.wconvT_bf16, a.wa_bf16, a.waT_bf16, a.ba, a.qv = _p(ops["wconvT"]), _p(ops["wa"]), _p(ops["waT"]), _p(ops["ba"]), _p(ops["qv"])
        a.p_drop, a.seed = m["p_drop"], m["seed"]
        a.Xp_bf16, a.Y_bf16, a.w, a.dout = _p(Xp), _p(Y), _p(w), _p(dout)
        a.dWconv_ext, a.dWa_ext, a.dqv, a.demb = _p(dWc), _p(dWa), _p(dqv), _p(demb)
        a.workspace, a.workspace_bytes = _p(ws), ws_bytes
        check(lib.nr_cnn_encoder_bwd(C.byref(a), _stream()), "nr_cnn_encoder_bwd")
        gWc = dWc[:, :, :d].permute(1, 0, 2).unsqueeze(1).contiguous()   # (F, 1, w, d)
        gbc = dWc[(win - 1) // 2, :, d].contiguous()                      # the tap of shift 0 reads the ones column
        return (None, demb, gWc, gbc, dWa[:, :Fn].contiguous(), dWa[:, Fn].contiguous(), dqv, None, None, None, None, None)


class LinearRowsFn(torch.autograd.Function):
    """y = act(x W^T + b) over dense fp32 rows x (n, K) -> (n, N); reference: nn.Linear (TANR/__init__.py:58-61)."""

    @staticmethod
    def forward(ctx, x, W, b, relu, cache, prefix):
        lib = load_library()
        dev = require_cuda()
        n, K = x.shape
        N = W.shape[0]
        ldx, ldn = ru8(K + 1), ru8(N + 1)
        ops = cache.get(prefix, (W, b), lambda W, b: dict(w=cast_pad(W, ldx), wT=cast_pad(W, ldn, transpose=True),
                                                         b=b.float().contiguous()))
        xs = x.float()
        X = torch.empty((n, ldx), dtype=torch.bfloat16, device=dev)
        ld_out = (N + 3) // 4 * 4
        out = torch.empty((n, ld_out), dtype=torch.float32, device=dev)
        check(lib.nr_linear_rows_fwd(_p(xs), n, K, xs.stride(0), xs.stride(1), _p(X), ldx, _p(ops["w"]), N, ldx, _p(ops["b"]),
                                     int(relu), _p(out), ld_out, _stream()), "nr_linear_rows_fwd")
        ctx.save_for_backward(X, out if relu else torch.empty(0, device=dev))
        ctx.meta = dict(n=n, K=K, N=N, relu=bool(relu), ops=ops, ld_out=ld_out, need_dx=x.requires_grad)
        return out[:, :N]

    @staticmethod
    def backward(ctx, dy):
        lib = load_library()
        X, out = ctx.saved_tensors
        m = ctx.meta
        n, K, N, ops = m["n"], m["K"], m["N"], m["ops"]
        dev = X.device
        ldx, ldn = ru8(K + 1), ru8(N + 1)
        g = torch.zeros((n, m["ld_out"]), dtype=torch.float32, device=dev)
        g[:, :N] = dy
        dY = torch.empty((n, ldn), dtype=torch.bfloat16, device=dev)
        dW = torch.zeros((N, ldx), dtype=torch.float32, device=dev)
        ld_dx = (K + 3) // 4 * 4
        dx = torch.empty((n, ld_dx), dtype=torch.float32, device=dev) if m["need_dx"] else None
        check(lib.nr_linear_rows_bwd(_p(g), _p(out) if m["relu"] else None, n, N, m["ld_out"], _p(dY), ldn, _p(X), K, ldx,
                                     _p(ops["wT"]), ldn, _p(dW), _p(dx), ld_dx, _stream()), "nr_linear_rows_bwd")
        return (dx[:, :K] if dx is not None else None), dW[:, :K].contiguous(), dW[:, K].contiguous(), None, None, None


class EmbeddingF32Fn(torch.autograd.Function):
    """fp32 table lookup with padding_idx=0 gradient semantics (LSTUR category / user embeddings)."""

    @staticmethod
    def forward(ctx, ids, table, bad_flag):
        lib = load_library()
        dev = require_cuda()
        ids = ids.contiguous().view(-1)
        V, D = table.shape
        tbl = table.float().contiguous()
        out = torch.empty((ids.numel(), D), dtype=torch.float32, device=dev)
        check(lib.nr_embedding_f32_fwd(_p(ids), ids.numel(), _p(tbl), V, D, _p(out), _p(bad_flag), _stream()), "nr_embedding_f32_fwd")
        ctx.save_for_backward(ids)
        ctx.shape = (V, D)
        return out

    @staticmethod
    def backward(ctx, dout):
        lib = load_library()
        (ids,) = ctx.saved_tensors
        V, D = ctx.shape
        dout = dout.contiguous().float()
        dt = torch.zeros((V, D), dtype=torch.float32, device=dout.device)
        check(lib.nr_embedding_f32_bwd(_p(ids), ids.numel(), _p(dout), V, D, _p(dt), _stream()), "nr_embedding_f32_bwd")
        return None, dt, None


class ElementEncoderFn(torch.autograd.Function):
    """relu(Linear(embedding(id)))  -- reference NAML/news_encoder.py:40-47."""

    @staticmethod
    def forward(ctx, ids, emb_w, W, b, cache, prefix, bad_flag):
        lib = load_library()
        dev = require_cuda()
        ids = ids.contiguous().view(-1)
        n = ids.numel()
        V, E = emb_w.shape
        Fn = W.shape[0]
        lde, ldf = ru8(E + 1), ru8(Fn + 1)
        ops = cache.get(prefix, (W, b), lambda W, b: dict(w=cast_pad(W, lde), wT=cast_pad(W, ldf, transpose=True),
                                                         b=b.float().contiguous()))
        table = table_operand(cache, prefix + ".table", emb_w)
        Eb = torch.empty((n, lde), dtype=torch.bfloat16, device=dev)
        out = torch.empty((n, Fn), dtype=torch.float32, device=dev)
        check(lib.nr_element_encoder_fwd(_p(ids), n, _p(table), V, E, lde, _p(Eb), _p(ops["w"]), Fn, _p(ops["b"]), _p(out),
                                         _p(bad_flag), _stream()), "nr_element_encoder_fwd")
        ctx.save_for_backward(ids, Eb, out)
        ctx.meta = dict(n=n, V=V, E=E, F=Fn, ops=ops)
        return out

    @staticmethod
    def backward(ctx, dout):
        lib = load_library()
        ids, Eb, out = ctx.saved_tensors
        m = ctx.meta
        n, V, E, Fn, ops = m["n"], m["V"], m["E"], m["F"], m["ops"]
        dev = Eb.device
        lde, ldf = ru8(E + 1), ru8(Fn + 1)
        dout = dout.contiguous().float()
        dY = torch.empty((n, ldf), dtype=torch.bfloat16, device=dev)
        dW = torch.zeros((Fn, lde), dtype=torch.float32, device=dev)
        dt = torch.zeros((V, E), dtype=torch.float32, device=dev)
        check(lib.nr_element_encoder_bwd(_p(ids), n, _p(dout), _p(out), Fn, _p(dY), ldf, _p(Eb), E, lde, _p(ops["wT"]), _p(dW),
                                         _p(dt), V, _stream()), "nr_element_encoder_bwd")
        return None, dt, dW[:, :E].contiguous(), dW[:, E].contiguous(), None, None, None
