"""torch.autograd.Function wrappers over the C ABI.

Each Function allocates its buffers with torch (the caller owns every buffer, see the header), passes raw
device pointers + the current CUDA stream to one composite C call, and returns torch tensors.  No
arithmetic happens here; `torch.cat`/slicing of parameters is layout plumbing only.
"""
from __future__ import annotations

import ctypes as C
import numbers
import os

import torch

from . import (MhsaEncoderBwdArgs, MhsaEncoderFwdArgs, NewsrecError, check, load_library, require_cuda)


def ru8(x: int) -> int:
    return (x + 7) // 8 * 8


def ru16(x: int) -> int:
    return (x + 15) // 16 * 16


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


# Data-parallel hook (ddp.FlatGradients): the gradient view of the embedding table carries, under this attribute, the owning
# buffer's {"event": torch.cuda.Event, "recorded": bool}; the news-encoder backward that writes that view records the event as
# soon as the embedding gradient is complete, so that its all-reduce can start under the remaining backward kernels.  Keyed by the
# gradient storage, so that models with a FlatGradients each (an ensemble) record into their own buffer's event.
GRAD_READY_ATTR = "_newsrec_grad_ready"

_seed_counter = [0x243F6A8885A308D3]


def _seed_from(counter: int) -> int:
    return (counter ^ (torch.initial_seed() & 0xFFFFFFFFFFFFFFFF) ^ (int(os.environ.get("RANK", "0")) << 48)) & 0xFFFFFFFFFFFFFFFF


def next_seed() -> int:
    """Per-call dropout seed (counter based, mixed with torch's CPU seed so manual_seed() reproduces runs)."""
    _seed_counter[0] = (_seed_counter[0] * 6364136223846793005 + 1442695040888963407) & 0xFFFFFFFFFFFFFFFF
    return _seed_from(_seed_counter[0])


def peek_seeds(n: int = 1):
    """The next `n` values next_seed() will return, without advancing the counter (tests hand them to the oracle so
    that it applies exactly the masks the kernels are going to draw)."""
    c, out = _seed_counter[0], []
    for _ in range(n):
        c = (c * 6364136223846793005 + 1442695040888963407) & 0xFFFFFFFFFFFFFFFF
        out.append(_seed_from(c))
    return out


# ---------------------------------------------------------------------------------------------------
# bf16 operand cache: fp32 nn.Parameters -> padded bf16 tensor-core operands, rebuilt only when a
# parameter's version counter (bumped by optimizer.step / load_state_dict) or storage changes.
# ---------------------------------------------------------------------------------------------------
class OperandCache:
    def __init__(self):
        self._store = {}

    def get(self, name, params, builder):
        key = tuple((p.data_ptr(), p._version, tuple(p.shape)) for p in params)
        hit = self._store.get(name)
        if hit is not None and hit[0] == key:
            return hit[1]
        with torch.no_grad():
            val = builder(*[p.detach() for p in params])
        self._store[name] = (key, val)
        return val

    def clear(self):
        self._store.clear()

    def invalidate_operands(self):
        """Drop every entry derived from parameters (what an optimizer step does implicitly by bumping their version
        counters); parameter-independent workspaces stay.  bench.py calls it every step so that the timed step pays for
        the operand refresh of real training."""
        for name in [n for n, (key, _) in self._store.items() if key]:
            del self._store[name]


DIRECT_GRAD_MARK = "_newsrec_direct_grad"


def grad_sink(p):
    """The parameter's own gradient storage if the kernels may accumulate into it directly, else None.
    Direct accumulation bypasses AccumulateGrad (tensor / DDP hooks do not fire, torch.autograd.grad returns nothing for the
    parameter), so it is an explicit opt-in: the owner of the gradient storage marks it (ddp.FlatGradients does); a .grad that
    merely exists -- e.g. after optimizer.zero_grad(set_to_none=False) -- takes the ordinary return path."""
    g = getattr(p, "grad", None)
    if g is None or not getattr(g, DIRECT_GRAD_MARK, False):
        return None
    if not p.requires_grad or g.dtype != torch.float32 or not g.is_contiguous() or g.device != p.device \
            or g.shape != p.shape or g.data_ptr() % 16 != 0:  # 16-byte vector reductions (red.global.add.v4.f32)
        return None
    return g


def cast_pad(src: torch.Tensor, ld: int, transpose: bool = False) -> torch.Tensor:
    """fp32 [R][C] -> zero padded bf16 [R][ld] (or the transpose [C][ld]) on the device."""
    lib = load_library()
    src = src.contiguous().float()
    R, Cc = src.shape
    rows = Cc if transpose else R
    dst = torch.empty((rows, ld), dtype=torch.bfloat16, device=src.device)
    check(lib.nr_cast_pad_bf16(_p(src), R, Cc, Cc, _p(dst), ld, int(transpose), _stream()), "nr_cast_pad_bf16")
    return dst


def precision_mode(config):
    """"fast" | "accurate" from a model config (config.py: precision)."""
    if bool(getattr(config, "fused_news_encoder", False)):
        raise NewsrecError("config.fused_news_encoder: the one-kernel news front end no longer exists; precision='accurate' "
                           "has the same storage contract")
    mode = str(getattr(config, "precision", "fast"))
    if mode not in ("fast", "accurate"):
        raise NewsrecError(f"config.precision must be 'fast' or 'accurate' (got {mode!r})")
    return mode


def qkv_pitches(d):
    """(sec, ld3) of the projected rows Q | K | V: sections at columns 0, sec, 2*sec with sec = round_up(d, 8) so that every
    section has the same 16-byte phase (abi.cu qkv_section); row pitch ld3 = round_up(3*sec, 16)."""
    sec = ru8(d)
    return sec, ru16(3 * sec)


def stack_qkv(mq, mk, mv):
    """W_Q | W_K | W_V (or the biases) stacked on dim 0 with zero rows up to the section stride after each."""
    d = mq.shape[0]
    pad = qkv_pitches(d)[0] - d
    parts = []
    for m in (mq, mk, mv):
        m = m.float()
        parts.append(m)
        if pad:
            parts.append(m.new_zeros((pad,) + tuple(m.shape[1:])))
    return torch.cat(parts, dim=0)


def cast_pad_many(specs):
    """[(fp32 [R][C] tensor, ld, transpose), ...] (at most 8) -> the zero padded bf16 operands, ONE launch for all of them."""
    lib = load_library()
    n = len(specs)
    srcs = [t.contiguous().float() for t, _, _ in specs]
    dsts = [torch.empty(((s.shape[1] if tr else s.shape[0]), ld), dtype=torch.bfloat16, device=s.device) for s, (_, ld, tr) in zip(srcs, specs)]
    arr_i = lambda vals: (C.c_int * n)(*vals)
    check(lib.nr_cast_pad_bf16_many(n, (C.c_void_p * n)(*[s.data_ptr() for s in srcs]), arr_i([s.shape[0] for s in srcs]),
                                    arr_i([s.shape[1] for s in srcs]), arr_i([s.shape[1] for s in srcs]),
                                    (C.c_void_p * n)(*[t.data_ptr() for t in dsts]), arr_i([ld for _, ld, _ in specs]),
                                    arr_i([int(tr) for _, _, tr in specs]), _stream()), "nr_cast_pad_bf16_many")
    return dsts


def mhsa_operands(cache: OperandCache, prefix, Wq, bq, Wk, bk, Wv, bv, Wa, ba, qv):
    d, q = Wq.shape[0], Wa.shape[0]
    ldx, ldq = ru8(d + 1), ru16(q)
    ld3 = qkv_pitches(d)[1]

    def build(Wq, bq, Wk, bk, Wv, bv, Wa, ba, qv):
        wqkv = stack_qkv(Wq, Wk, Wv)
        w, wT, wa, waT = cast_pad_many([(wqkv, ldx, False), (wqkv, ld3, True), (Wa, ldx, False), (Wa, ldq, True)])
        return dict(wqkv=w, wqkvT=wT, bqkv=stack_qkv(bq, bk, bv).contiguous(), wa=wa, waT=waT,
                    ba=ba.float().contiguous(), qv=qv.float().contiguous())

    return cache.get(prefix, (Wq, bq, Wk, bk, Wv, bv, Wa, ba, qv), build)


def table_operand(cache: OperandCache, name, weight):
    ldx = ru8(weight.shape[1] + 1)
    return cache.get(name, (weight,), lambda w: cast_pad(w, ldx))


# ---------------------------------------------------------------------------------------------------
# NRMS NewsEncoder / UserEncoder: gather|dense -> MHSA -> additive pooling in ONE C call each way
# ---------------------------------------------------------------------------------------------------
class MhsaPoolEncoderFn(torch.autograd.Function):
    """forward(ids|None, dense|None, emb_weight|None, Wq,bq,Wk,bk,Wv,bv, Wa,ba,qv, heads, p_drop, cache, prefix, bad_flag,
               precise, pos|None)

    ids   : int64 (n_seq, T) device tensor  (news encoder)   -- reference src/model/NRMS/news_encoder.py:27-48
    dense : fp32  (n_seq, T, d) any strides (user encoder)   -- reference src/model/NRMS/user_encoder.py:15-26
    pos   : fp32  (T, d) added to every sequence of `dense` before the projection (reference src/model/Exp1/user_encoder.py:
            26-27); its gradient is the input gradient summed over the sequences
    """

    @staticmethod
    def forward(ctx, ids, dense, emb_w, Wq, bq, Wk, bk, Wv, bv, Wa, ba, qv, heads, p_drop, cache, prefix, bad_flag, precise=False,
                pos=None):
        lib = load_library()
        dev = require_cuda()
        d, q = Wq.shape[0], Wa.shape[0]
        ldx = ru8(d + 1)
        sec, ld3 = qkv_pitches(d)
        ops = mhsa_operands(cache, prefix, Wq, bq, Wk, bk, Wv, bv, Wa, ba, qv)
        a = MhsaEncoderFwdArgs()
        if ids is not None:
            n_seq, T = ids.shape
            ids = ids.contiguous()
            table = table_operand(cache, prefix + ".table", emb_w)
            a.ids, a.table_bf16, a.V = _p(ids), _p(table), emb_w.shape[0]
            a.dense = None
        else:
            n_seq, T, dd = dense.shape
            if dd != d:
                raise NewsrecError(f"user encoder input width {dd} != model width {d}")
            dense = dense.float()
            a.ids, a.table_bf16, a.V = None, None, 0
            a.dense = _p(dense)
            a.dense_s_seq, a.dense_s_tok, a.dense_s_col = dense.stride()
            table = None
        if pos is not None:
            if ids is not None:
                raise NewsrecError("a positional addend applies to the dense (user-level) input only")
            if tuple(pos.shape) != (T, d):
                raise NewsrecError(f"positional addend of shape {tuple(pos.shape)} for inputs of {T} positions x {d}")
            a.dense_pos = _p(pos.detach().float().contiguous())
        n_tok = n_seq * T
        need_bwd = any(ctx.needs_input_grad)
        # precision modes (config.precision, DESIGN.md section 4):
        #   "fast"      bf16 storage of every activation (Q|K|V, probabilities, context): fastest, ~6e-3 from the fp32 result
        #   "accurate"  V / probabilities / context as hi/lo bf16 pairs on the same unfused kernels + fp32-accurate user
        #               encoder: within the blueprint's 1e-3 of the fp32 oracle on bf16-rounded weights
        mode = precise if isinstance(precise, str) else ("accurate" if precise else "fast")
        accurate = ids is not None and mode == "accurate" and bool(lib.nr_mhsa_accurate_supported(T, d, heads))
        precise_dense = ids is None and mode == "accurate"  # user encoder: fp32-accurate forward (abi.cu)
        X = QKV = C_lo = V_lo = None
        X = torch.empty((n_tok, ldx), dtype=torch.bfloat16, device=dev)
        if not precise_dense:  # the precise dense path keeps no bf16 Q|K|V; its backward recomputes it from X
            QKV = torch.empty((n_tok, ld3), dtype=torch.bfloat16, device=dev)
        Cx = torch.empty((n_tok, ldx), dtype=torch.bfloat16, device=dev)
        w = torch.empty((n_tok,), dtype=torch.float32, device=dev)
        out = torch.empty((n_seq, d), dtype=torch.float32, device=dev)
        seed = next_seed() if p_drop > 0 else 0
        a.n_seq, a.T, a.d, a.heads, a.q, a.ldx, a.ld3 = n_seq, T, d, heads, q, ldx, ld3
        a.wqkv_bf16, a.bqkv, a.wa_bf16, a.ba, a.qv = _p(ops["wqkv"]), _p(ops["bqkv"]), _p(ops["wa"]), _p(ops["ba"]), _p(ops["qv"])
        a.p_drop, a.seed = float(p_drop), seed
        if accurate:
            C_lo = torch.empty((n_tok, ldx), dtype=torch.bfloat16, device=dev)
            V_lo = torch.empty((n_tok, sec), dtype=torch.bfloat16, device=dev)
            a.C_lo_bf16, a.V_lo_bf16 = _p(C_lo), _p(V_lo)
        keep = None
        if precise_dense:
            kcat = cache.get(prefix + ".kcat", (Wq, Wk, Wv), lambda Wq, Wk, Wv: cast_pad(
                torch.cat((torch.nn.functional.pad(stack_qkv(Wq, Wk, Wv), (0, ldx - d)),) * 2, dim=1), 2 * ldx))
            C_lo = torch.empty((n_tok, ldx), dtype=torch.bfloat16, device=dev)
            keep = (torch.empty((n_tok, 2 * ldx), dtype=torch.bfloat16, device=dev), torch.empty((n_tok, 3 * sec), dtype=torch.float32, device=dev))
            a.wqkv_kcat_bf16, a.X_kcat_bf16, a.QKV_f32, a.C_lo_bf16 = _p(kcat), _p(keep[0]), _p(keep[1]), _p(C_lo)
        a.X_bf16, a.QKV_bf16, a.C_bf16, a.w, a.out = _p(X), _p(QKV), _p(Cx), _p(w), _p(out)
        a.bad_id_flag = _p(bad_flag)
        check(lib.nr_mhsa_encoder_fwd(C.byref(a), _stream()), "nr_mhsa_encoder_fwd")
        if need_bwd:
            ctx.save_for_backward(X, QKV if QKV is not None else torch.empty(0, device=dev), Cx, w,
                                  ids if ids is not None else torch.empty(0, device=dev))
        ctx.meta = dict(n_seq=n_seq, T=T, d=d, q=q, heads=heads, p_drop=float(p_drop), seed=seed, ops=ops,
                        has_ids=ids is not None, V=emb_w.shape[0] if ids is not None else 0,
                        dense_shape=None if dense is None else tuple(dense.shape),
                        params=(emb_w, Wq, bq, Wk, bk, Wv, bv, Wa, ba, qv), cache=cache, prefix=prefix,
                        pos=pos, table=table)
        return out

    @staticmethod
    def backward(ctx, dout):
        lib = load_library()
        X, QKV, Cx, w, ids = ctx.saved_tensors
        m = ctx.meta
        dev = X.device
        d, q, T, n_seq = m["d"], m["q"], m["T"], m["n_seq"]
        ldx, ldq = ru8(d + 1), ru16(q)
        sec, ld3 = qkv_pitches(d)
        ops = m["ops"]
        dout = dout.contiguous().float()
        emb_w, Wq, bq, Wk, bk, Wv, bv, Wa, ba, qv = m["params"]
        # Parameters whose .grad storage is marked for direct accumulation (ddp.FlatGradients; see grad_sink) are
        # accumulated IN PLACE by the kernels and get None from this Function: no zero fill, no slice
        # copies, no AccumulateGrad adds (together ~50 small framework kernels and 3 passes over the 85 MB embedding
        # gradient per step).  Anything else takes the allocate-and-return path.
        sinks = [grad_sink(t) for t in (Wq, bq, Wk, bk, Wv, bv, Wa, ba, qv)]
        direct = all(g is not None for g in sinks)
        if direct:
            ws_grads = m["cache"].get(m["prefix"] + ".grad_ws", (), lambda: dict(
                dWqkv=torch.zeros((3 * sec, ldx), dtype=torch.float32, device=dev),
                dWa=torch.zeros((q, ldx), dtype=torch.float32, device=dev)))
            dWqkv, dWa, dqv = ws_grads["dWqkv"], ws_grads["dWa"], sinks[8]
        else:
            dWqkv = torch.zeros((3 * sec, ldx), dtype=torch.float32, device=dev)
            dWa = torch.zeros((q, ldx), dtype=torch.float32, device=dev)
            dqv = torch.zeros((q,), dtype=torch.float32, device=dev)
        demb = ddense = None
        emb_direct = False
        if m["has_ids"]:
            demb = grad_sink(emb_w)
            emb_direct = demb is not None
            if not emb_direct:
                demb = torch.zeros((m["V"], d), dtype=torch.float32, device=dev)
        else:
            ddense = torch.empty((n_seq * T, d), dtype=torch.float32, device=dev)
        dpos, pos_direct = None, False
        if m["pos"] is not None:  # the kernel adds into dpos: the parameter's own gradient storage, or a zeroed buffer returned below
            dpos = grad_sink(m["pos"])
            pos_direct = dpos is not None
            if not pos_direct:
                dpos = torch.zeros((T, d), dtype=torch.float32, device=dev)
        ws_bytes = int(lib.nr_mhsa_encoder_bwd_workspace(n_seq, T, d, q))
        ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
        a = MhsaEncoderBwdArgs()
        a.n_seq, a.T, a.d, a.heads, a.q, a.ldx, a.ld3, a.ldq = n_seq, T, d, m["heads"], q, ldx, ld3, ldq
        a.ids = _p(ids) if m["has_ids"] else None
        a.V = m["V"]
        a.table_bf16 = _p(m["table"]) if m["has_ids"] else None  # the forward's table: its row 0 decides which tokens are live
        a.wqkvT_bf16, a.wa_bf16, a.waT_bf16, a.ba, a.qv = _p(ops["wqkvT"]), _p(ops["wa"]), _p(ops["waT"]), _p(ops["ba"]), _p(ops["qv"])
        a.p_drop, a.seed = m["p_drop"], m["seed"]
        a.X_bf16, a.QKV_bf16, a.C_bf16, a.w, a.dout = _p(X), (_p(QKV) if QKV.numel() else None), _p(Cx), _p(w), _p(dout)
        a.wqkv_bf16, a.bqkv = _p(ops["wqkv"]), _p(ops["bqkv"])
        hook = getattr(demb, GRAD_READY_ATTR, None) if (m["has_ids"] and emb_direct) else None
        if hook is not None:
            a.emb_grad_ready_event = C.c_void_p(hook["event"].cuda_event)
            hook["recorded"] = True
        a.dWqkv_ext, a.dWa_ext, a.dqv = _p(dWqkv), _p(dWa), _p(dqv)
        a.demb, a.ddense, a.dpos = _p(demb), _p(ddense), _p(dpos)
        a.workspace, a.workspace_bytes = _p(ws), ws_bytes
        check(lib.nr_mhsa_encoder_bwd(C.byref(a), _stream()), "nr_mhsa_encoder_bwd")
        g_dense = ddense.view(m["dense_shape"]) if ddense is not None else None
        g_emb = None if emb_direct else demb
        g_pos = None if pos_direct else dpos
        if direct:
            for i in range(3):
                check(lib.nr_accumulate_ext_grad(_p(dWqkv[i * sec:i * sec + d]), d, ldx, d, _p(sinks[2 * i]), _p(sinks[2 * i + 1]),
                                                 _stream()), "nr_accumulate_ext_grad")
            check(lib.nr_accumulate_ext_grad(_p(dWa), q, ldx, d, _p(sinks[6]), _p(sinks[7]), _stream()), "nr_accumulate_ext_grad")
            return (None, g_dense, g_emb) + (None,) * 15 + (g_pos,)
        gW = [dWqkv[i * sec:i * sec + d, :d].contiguous() for i in range(3)]
        gb = [dWqkv[i * sec:i * sec + d, d].contiguous() for i in range(3)]
        return (None, g_dense, g_emb, gW[0], gb[0], gW[1], gb[1], gW[2], gb[2],
                dWa[:, :d].contiguous(), dWa[:, d].contiguous(), dqv, None, None, None, None, None, None, g_pos)


# ---------------------------------------------------------------------------------------------------
# AdditiveAttention over dense fp32 rows (NAML / TANR user encoder, NAML 4-view fusion, standalone module)
# ---------------------------------------------------------------------------------------------------
class AdditiveAttentionFn(torch.autograd.Function):
    """reference src/model/general/attention/additive.py:27-53;  x (N, S, D) fp32 -> (N, D).
    precision "fast": x enters as bf16 rows; "accurate": as a hi/lo bf16 pair (the scores read the hi plane, the pooled sum
    both: ~16 mantissa bits); the backward reads the hi plane in both modes."""

    @staticmethod
    def forward(ctx, x, Wa, ba, qv, cache, prefix, precision="fast"):
        lib = load_library()
        dev = require_cuda()
        if precision not in ("fast", "accurate"):
            raise NewsrecError(f"additive attention precision must be 'fast' or 'accurate' (got {precision!r})")
        N, S, D = x.shape
        q = Wa.shape[0]
        ldx, ldq = ru8(D + 1), ru16(q)
        ops = cache.get(prefix, (Wa, ba, qv), lambda Wa, ba, qv: dict(
            wa=cast_pad(Wa, ldx), waT=cast_pad(Wa, ldq, transpose=True), ba=ba.float().contiguous(),
            qv=qv.float().contiguous()))
        xf = x.float()
        X = torch.empty((N * S, ldx), dtype=torch.bfloat16, device=dev)
        xs = xf.reshape(N * S, D) if xf.is_contiguous() else xf.contiguous().view(N * S, D)
        out = torch.empty((N, D), dtype=torch.float32, device=dev)
        w = torch.empty((N * S,), dtype=torch.float32, device=dev)
        if precision == "accurate":
            X_lo = torch.empty((N * S, ldx), dtype=torch.bfloat16, device=dev)
            check(lib.nr_rows_to_bf16_hilo(_p(xs), N * S, D, xs.stride(0), xs.stride(1), _p(X), _p(X_lo), ldx, _stream()),
                  "nr_rows_to_bf16_hilo")
            check(lib.nr_additive_attention_fwd_hilo(_p(X), _p(X_lo), N, S, D, ldx, _p(ops["wa"]), q, ldx, _p(ops["ba"]),
                                                     _p(ops["qv"]), _p(out), D, _p(w), _stream()), "nr_additive_attention_fwd_hilo")
        else:
            check(lib.nr_rows_to_bf16(_p(xs), N * S, D, xs.stride(0), xs.stride(1), _p(X), ldx, _stream()), "nr_rows_to_bf16")
            check(lib.nr_additive_attention_fwd(_p(X), N, S, D, ldx, _p(ops["wa"]), q, ldx, _p(ops["ba"]), _p(ops["qv"]),
                                                _p(out), D, _p(w), _stream()), "nr_additive_attention_fwd")
        ctx.save_for_backward(X, w)
        ctx.meta = dict(N=N, S=S, D=D, q=q, ops=ops)
        return out

    @staticmethod
    def backward(ctx, dout):
        lib = load_library()
        X, w = ctx.saved_tensors
        m = ctx.meta
        N, S, D, q, ops = m["N"], m["S"], m["D"], m["q"], m["ops"]
        dev = X.device
        ldx, ldq = ru8(D + 1), ru16(q)
        dout = dout.contiguous().float()
        dX = torch.empty((N * S, ldx), dtype=torch.bfloat16, device=dev)
        dWa = torch.zeros((q, ldx), dtype=torch.float32, device=dev)
        dqv = torch.zeros((q,), dtype=torch.float32, device=dev)
        ws_bytes = int(lib.nr_additive_attention_bwd_workspace(N, S, q))
        ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
        check(lib.nr_additive_attention_bwd(_p(X), N, S, D, ldx, _p(ops["wa"]), _p(ops["waT"]), q, ldx, ldq, _p(ops["ba"]),
                                            _p(ops["qv"]), _p(w), _p(dout), D, _p(dX), ldx, _p(dWa), _p(dqv), _p(ws),
                                            ws_bytes, _stream()), "nr_additive_attention_bwd")
        gx = dX[:, :D].float().view(N, S, D)
        return gx, dWa[:, :D].contiguous(), dWa[:, D].contiguous(), dqv, None, None, None


# ---------------------------------------------------------------------------------------------------
# DotProductClickPredictor
# ---------------------------------------------------------------------------------------------------
class DotScoreFn(torch.autograd.Function):
    """reference src/model/general/click_predictor/dot_product.py:8-19;  (B,C,D),(B,D) -> (B,C) logits."""

    @staticmethod
    def forward(ctx, cand, user):
        lib = load_library()
        dev = require_cuda()
        cand = cand.contiguous().float()
        user = user.contiguous().float()
        B, Cn, D = cand.shape
        logits = torch.empty((B, Cn), dtype=torch.float32, device=dev)
        check(lib.nr_dot_score_fwd(_p(cand), _p(user), B, Cn, D, _p(logits), _stream()), "nr_dot_score_fwd")
        ctx.save_for_backward(cand, user)
        return logits

    @staticmethod
    def backward(ctx, dlogits):
        lib = load_library()
        cand, user = ctx.saved_tensors
        B, Cn, D = cand.shape
        dlogits = dlogits.contiguous().float()
        dcand = torch.empty_like(cand)
        duser = torch.empty_like(user)
        check(lib.nr_dot_score_bwd(_p(cand), _p(user), _p(dlogits), B, Cn, D, _p(dcand), _p(duser), _stream()),
              "nr_dot_score_bwd")
        return dcand, duser


# ---------------------------------------------------------------------------------------------------
# standalone MultiHeadSelfAttention (projection + attention core, no pooling)
# ---------------------------------------------------------------------------------------------------
class MhsaFn(torch.autograd.Function):
    """reference src/model/general/attention/multihead_self.py:46-76 with Q=K=V=x, length=None."""

    @staticmethod
    def forward(ctx, x, Wq, bq, Wk, bk, Wv, bv, heads, cache, prefix):
        lib = load_library()
        dev = require_cuda()
        N, T, d = x.shape
        ldx, ld3 = ru8(d + 1), ru16(3 * d)

        def build(Wq, bq, Wk, bk, Wv, bv):
            wqkv = torch.cat((Wq, Wk, Wv), dim=0)
            return dict(wqkv=cast_pad(wqkv, ldx), wqkvT=cast_pad(wqkv, ld3, transpose=True),
                        bqkv=torch.cat((bq, bk, bv)).float().contiguous())

        ops = cache.get(prefix, (Wq, bq, Wk, bk, Wv, bv), build)
        xs = x.float().contiguous().view(N * T, d)
        X = torch.empty((N * T, ldx), dtype=torch.bfloat16, device=dev)
        check(lib.nr_rows_to_bf16(_p(xs), N * T, d, d, 1, _p(X), ldx, _stream()), "nr_rows_to_bf16")
        QKV = torch.empty((N * T, ld3), dtype=torch.bfloat16, device=dev)
        check(lib.nr_linear(_p(X), N * T, ldx, _p(ops["wqkv"]), 3 * d, ldx, d, 1, 0, 128, _p(ops["bqkv"]), 0, _p(QKV), ld3, 1,
                            _stream()), "nr_linear")
        Cx = torch.empty((N * T, ldx), dtype=torch.bfloat16, device=dev)
        check(lib.nr_mhsa_core_fwd(_p(QKV), ld3, d, N, T, heads, d // heads, _p(Cx), ldx, 0.0, 0, _stream()), "nr_mhsa_core_fwd")
        ctx.save_for_backward(X, QKV)
        ctx.meta = dict(N=N, T=T, d=d, heads=heads, ops=ops)
        return Cx[:, :d].float().view(N, T, d)

    @staticmethod
    def backward(ctx, dctx):
        lib = load_library()
        X, QKV = ctx.saved_tensors
        m = ctx.meta
        N, T, d, heads, ops = m["N"], m["T"], m["d"], m["heads"], m["ops"]
        dev = X.device
        ldx, ld3 = ru8(d + 1), ru16(3 * d)
        g = dctx.float().contiguous().view(N * T, d)
        dC = torch.empty((N * T, ldx), dtype=torch.bfloat16, device=dev)
        check(lib.nr_rows_to_bf16(_p(g), N * T, d, d, 1, _p(dC), ldx, _stream()), "nr_rows_to_bf16")
        dQKV = torch.empty((N * T, ld3), dtype=torch.bfloat16, device=dev)
        check(lib.nr_mhsa_core_bwd(_p(QKV), ld3, d, _p(dC), ldx, N, T, heads, d // heads, _p(dQKV), ld3, _stream()),
              "nr_mhsa_core_bwd")
        dW = torch.zeros((3 * d, ldx), dtype=torch.float32, device=dev)
        for c0 in range(0, d + 1, 512):  # nr_gemm_tn takes at most 512 columns of [X | 1] per launch
            check(lib.nr_gemm_tn(_p(dQKV), N * T, 3 * d, ld3, _p(X), N * T, d + 1, ldx, c0, min(512, d + 1 - c0), 0, _p(dW[:, c0:]),
                                 ldx, _stream()), "nr_gemm_tn")
        dx = torch.empty((N * T, d), dtype=torch.float32, device=dev)
        check(lib.nr_linear(_p(dQKV), N * T, ld3, _p(ops["wqkvT"]), d, ld3, 3 * d, 1, 0, 128, None, 0, _p(dx), d, 0, _stream()),
              "nr_linear")
        gW = [dW[i * d:(i + 1) * d, :d].contiguous() for i in range(3)]
        gb = [dW[i * d:(i + 1) * d, d].contiguous() for i in range(3)]
        return dx.view(N, T, d), gW[0], gb[0], gW[1], gb[1], gW[2], gb[2], None, None, None


# ---------------------------------------------------------------------------------------------------
# Batched scoring for evaluation (the "next" row N2 of SURVEY.md 8f)
# ---------------------------------------------------------------------------------------------------
def predict_impressions(news_matrix, cand_index, seg_offsets, user_vectors):
    """Scores of MANY impressions in one launch: reference src/evaluate.py:245-265 runs `get_prediction` once per impression
    and synchronises on `.tolist()` after each.  news_matrix (n_news, D) fp32 device matrix of news vectors (row = news
    index, instead of the evaluator's dict of rows), cand_index (n_cand,) int64 rows of the candidates of all impressions
    back to back, seg_offsets (n_impressions + 1,) int64 with seg_offsets[0] = 0, user_vectors (n_impressions, D).
    Returns (n_cand,) fp32 scores; candidate i of impression s is scores[seg_offsets[s] + i]."""
    lib = load_library()
    dev = require_cuda()
    news_matrix = news_matrix.to(dev).float().contiguous()
    user_vectors = user_vectors.to(dev).float().contiguous()
    cand_index = cand_index.to(dev).long().contiguous()
    seg_offsets = seg_offsets.to(dev).long().contiguous()
    n_seg = seg_offsets.numel() - 1
    if user_vectors.shape[0] != n_seg or user_vectors.shape[1] != news_matrix.shape[1]:
        raise NewsrecError("predict_impressions: user_vectors must be (len(seg_offsets) - 1, D)")
    scores = torch.empty((cand_index.numel(),), dtype=torch.float32, device=dev)
    flag = torch.zeros(1, dtype=torch.int32, device=dev)
    check(lib.nr_segment_dot(_p(news_matrix), news_matrix.shape[0], news_matrix.shape[1], _p(cand_index), cand_index.numel(),
                             _p(seg_offsets), n_seg, _p(user_vectors), _p(scores), _p(flag), _stream()), "nr_segment_dot")
    return scores


def impression_metrics(scores, labels, seg_offsets):
    """{AUC, MRR, nDCG@5, nDCG@10} of every impression in one launch (nr_impression_metrics): reference src/evaluate.py
    runs sklearn's roc_auc_score and NumPy's mrr / nDCG once per impression in a process pool.  scores (n_cand,) fp32,
    labels (n_cand,) 0/1, seg_offsets (n_impressions + 1,) int64 with seg_offsets[0] = 0.  Returns the (n_impressions, 4)
    fp64 device tensor; rows are NaN where the reference's metrics are undefined (include/newsrec_b200.h).  Raises
    ValueError if a label is not 0 or 1 (reads the device flag: one synchronisation)."""
    lib = load_library()
    dev = require_cuda()
    scores = scores.to(dev).float().contiguous()
    labels = labels.to(dev)
    if labels.dtype != torch.uint8:  # any value outside 0..255 must still reach the kernel as "not 0 / 1"
        labels = torch.where((labels >= 0) & (labels <= 1), labels, 2).to(torch.uint8)
    labels = labels.contiguous()
    seg_offsets = seg_offsets.to(dev).long().contiguous()
    if labels.numel() != scores.numel() or seg_offsets.dim() != 1 or seg_offsets.numel() < 1:
        raise NewsrecError("impression_metrics: labels must match scores; seg_offsets must be (n_impressions + 1,)")
    n_seg = seg_offsets.numel() - 1
    metrics = torch.empty((n_seg, 4), dtype=torch.float64, device=dev)
    if n_seg == 0:
        return metrics
    flag = torch.zeros(1, dtype=torch.int32, device=dev)
    check(lib.nr_impression_metrics(_p(scores), _p(labels), _p(seg_offsets), n_seg, _p(metrics), _p(flag), _stream()),
          "nr_impression_metrics")
    if int(flag.item()):
        raise ValueError("impression_metrics: a label is neither 0 nor 1")
    return metrics


def impression_ranks(scores, seg_offsets, bad_score_flag=None):
    """1-based rank of every candidate within its impression, one launch (nr_impression_ranks): ranks[i] = place_i + 1 with
    the place nr_impression_metrics uses (ties: the later candidate first; -0 == +0), so each impression's ranks are a
    permutation of 1..n.  scores (n_cand,) fp32, seg_offsets (n_impressions + 1,) int64.  Returns (n_cand,) int32 on the
    device.  An impression with a non-finite score sets bad_score_flag (a device int32 the caller checks); without one,
    a fresh flag is read here (one synchronisation) and ValueError raised."""
    lib = load_library()
    dev = require_cuda()
    scores = scores.to(dev).float().contiguous()
    seg_offsets = seg_offsets.to(dev).long().contiguous()
    if seg_offsets.dim() != 1 or seg_offsets.numel() < 1:
        raise NewsrecError("impression_ranks: seg_offsets must be (n_impressions + 1,)")
    ranks = torch.empty(scores.shape, dtype=torch.int32, device=dev)
    own = bad_score_flag is None
    flag = torch.zeros(1, dtype=torch.int32, device=dev) if own else bad_score_flag
    check(lib.nr_impression_ranks(_p(scores), _p(seg_offsets), seg_offsets.numel() - 1, _p(ranks), _p(flag), _stream()),
          "nr_impression_ranks")
    if own and int(flag.item()):
        raise ValueError("impression_ranks: an impression holds a non-finite score; its ranks are undefined")
    return ranks


def prediction_text(impression_ids, ranks, seg_offsets):
    """The prediction.txt bytes of many impressions, "<impression_id> [r1,r2,...,rn]\\n" per impression, as a (n_bytes,)
    uint8 device tensor: line lengths and their exclusive scan (nr_prediction_line_offsets, CUB in the library), one read of
    the total (a synchronisation), then one launch writing every line (nr_prediction_text).  impression_ids
    (n_impressions,) int64, non-negative; ranks (n_cand,) int32 from impression_ranks; seg_offsets as there."""
    lib = load_library()
    dev = require_cuda()
    ids = impression_ids.to(dev).long().contiguous()
    ranks = ranks.to(dev).int().contiguous()
    seg_offsets = seg_offsets.to(dev).long().contiguous()
    n_seg = seg_offsets.numel() - 1
    if ids.dim() != 1 or ids.numel() != n_seg:
        raise NewsrecError("prediction_text: impression_ids must be (len(seg_offsets) - 1,)")
    if n_seg == 0:
        return torch.empty(0, dtype=torch.uint8, device=dev)
    line_offsets = torch.empty(n_seg + 1, dtype=torch.int64, device=dev)
    ws_bytes = int(lib.nr_prediction_line_offsets_workspace(n_seg))
    if ws_bytes < 0:
        check(-1, "nr_prediction_line_offsets_workspace")
    workspace = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
    check(lib.nr_prediction_line_offsets(_p(ids), _p(ranks), _p(seg_offsets), n_seg, _p(line_offsets), _p(workspace), ws_bytes,
                                         _stream()), "nr_prediction_line_offsets")
    text = torch.empty(int(line_offsets[-1].item()), dtype=torch.uint8, device=dev)
    check(lib.nr_prediction_text(_p(ids), _p(ranks), _p(seg_offsets), n_seg, _p(line_offsets), _p(text), _stream()),
          "nr_prediction_text")
    return text


def top_k_scores(users, news, k, excl_rows=None, excl_offsets=None, *, categories=None, max_per_category=None):
    """The k best news of every user over the whole pool, one pass (nr_topk_dot): users (U, D) and news (n, D) fp32, scores
    users[u] . news[r] at fp32 level on the tensor cores (the bound is in include/newsrec_b200.h) without the U x n score
    matrix.  Optional exclusions in CSR form: user u never gets rows excl_rows[excl_offsets[u] .. excl_offsets[u + 1]).
    Returns (idx (U, k) int64, score (U, k) fp32) on the caller's stream, best first, equal scores by lower row; slots past
    the eligible news hold -1 / -inf.  Raises NewsrecError on bad arguments (before any launch), IndexError on an exclusion
    row outside [0, n) and ValueError on a non-finite score (both read device flags: one synchronisation).

    Diversified (nr_topk_dot_capped): with categories ((n,) integer keys, one per news row, any int32 value) and
    max_per_category = m, each list holds at most m news of one category: the pool is walked in the order above and a news is
    taken iff fewer than m taken news share its category and fewer than k are taken.  A user gets fewer than k news when the
    caps run out; m >= k gives the plain answer bit for bit.  The two arguments go together."""
    lib = load_library()
    if isinstance(k, bool) or not isinstance(k, int) or not 1 <= k <= 128:
        raise NewsrecError(f"top_k_scores: k={k!r} must be an integer in [1, 128]")
    if users.dim() != 2 or news.dim() != 2 or users.shape[1] != news.shape[1]:
        raise NewsrecError(f"top_k_scores: users {tuple(users.shape)} and news {tuple(news.shape)} must be (U, D) and (n, D)")
    if (excl_rows is None) != (excl_offsets is None):
        raise NewsrecError("top_k_scores: excl_rows and excl_offsets go together")
    capped = categories is not None or max_per_category is not None
    if capped:
        if categories is None or max_per_category is None:
            raise NewsrecError("top_k_scores: categories and max_per_category go together")
        if isinstance(max_per_category, bool) or not isinstance(max_per_category, numbers.Integral) or max_per_category < 1:
            raise NewsrecError(f"top_k_scores: max_per_category={max_per_category!r} must be an integer >= 1")
        max_per_category = min(int(max_per_category), k)  # a cap of k or more never binds
        categories = torch.as_tensor(categories)
        if categories.dim() != 1 or categories.shape[0] != news.shape[0]:
            raise NewsrecError(f"top_k_scores: categories {tuple(categories.shape)} must be (n,) = ({news.shape[0]},)")
        if categories.dtype.is_floating_point or categories.dtype.is_complex or categories.dtype == torch.bool:
            raise NewsrecError(f"top_k_scores: categories must hold integer keys, not {categories.dtype}")
        if categories.dtype != torch.int32 and categories.numel() and \
                (int(categories.min()) < -2 ** 31 or int(categories.max()) >= 2 ** 31):
            raise NewsrecError("top_k_scores: a category key does not fit in int32")
    dev = require_cuda()
    users = users.to(dev).float().contiguous()
    news = news.to(dev).float().contiguous()
    U, D = users.shape
    n = news.shape[0]
    if excl_offsets is not None:
        excl_offsets = excl_offsets.to(dev).long().contiguous()
        excl_rows = excl_rows.to(dev).long().contiguous()
        if excl_offsets.dim() != 1 or excl_offsets.numel() != U + 1 or excl_rows.dim() != 1:
            raise NewsrecError("top_k_scores: excl_offsets must be (U + 1,) and excl_rows 1-D")
        if excl_rows.numel() == 0:
            excl_rows = excl_rows.new_zeros(1)  # a valid address for an empty set
    ws_bytes = int(lib.nr_topk_dot_workspace(U, n, D, k))
    if ws_bytes < 0:
        check(-1, "nr_topk_dot_workspace")
    if U == 0 or n == 0:  # no user or nothing eligible: the library launches nothing
        return (torch.full((U, k), -1, dtype=torch.int64, device=dev),
                torch.full((U, k), float("-inf"), dtype=torch.float32, device=dev))
    idx = torch.empty((U, k), dtype=torch.int64, device=dev)
    score = torch.empty((U, k), dtype=torch.float32, device=dev)
    flags = torch.zeros(2, dtype=torch.int32, device=dev)
    workspace = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    if capped:
        cat = categories.to(device=dev, dtype=torch.int32).contiguous()
        check(lib.nr_topk_dot_capped(_p(users), U, D, _p(news), n, D, D, k, _p(excl_offsets), _p(excl_rows), _p(cat),
                                     max_per_category, _p(idx), _p(score), _p(flags[0:1]), _p(flags[1:2]), _p(workspace),
                                     ws_bytes, _stream()), "nr_topk_dot_capped")
    else:
        check(lib.nr_topk_dot(_p(users), U, D, _p(news), n, D, D, k, _p(excl_offsets), _p(excl_rows), _p(idx), _p(score),
                              _p(flags[0:1]), _p(flags[1:2]), _p(workspace), ws_bytes, _stream()), "nr_topk_dot")
    bad_row, bad_score = (int(x) for x in flags.tolist())
    if bad_row:
        raise IndexError("top_k_scores: an exclusion row is outside the news pool")
    if bad_score:
        raise ValueError("top_k_scores: a score is not finite; the order is undefined")
    return idx, score


POOL_RANK_MAX_TARGETS = 32  # targets per kernel row (nr_pool_ranks)


def target_parts(tgt_rows, tgt_offsets, excl_rows=None, excl_offsets=None, max_targets=POOL_RANK_MAX_TARGETS):
    """Host CSR plumbing of pool_ranks: query q with c > 0 targets becomes ceil(c / max_targets) kernel rows, each holding
    consecutive targets of q, so the kernel's targets are the caller's in the same order.  Each row excludes X_q and q's
    targets outside the row, so a rank does not depend on the split; a query without targets gets no row.  Returns
    (query (R,), offsets (R + 1,), excl_rows, excl_offsets (R + 1,)) as int64 NumPy arrays; offsets index tgt_rows."""
    import numpy as np
    tr, to = np.asarray(tgt_rows, np.int64), np.asarray(tgt_offsets, np.int64)
    counts = np.diff(to)
    nparts = (counts + max_targets - 1) // max_targets
    R = int(nparts.sum())
    query = np.repeat(np.arange(len(counts), dtype=np.int64), nparts)
    first = np.repeat(np.cumsum(nparts) - nparts, nparts)
    start = to[query] + max_targets * (np.arange(R, dtype=np.int64) - first)
    end = np.minimum(start + max_targets, to[query + 1])
    offsets = np.concatenate([start, end[-1:]]) if R else to[:1].copy()
    xlen = np.zeros(R, np.int64) if excl_offsets is None else \
        np.asarray(excl_offsets, np.int64)[query + 1] - np.asarray(excl_offsets, np.int64)[query]
    split = np.flatnonzero(nparts[query] > 1)
    extra = np.zeros(R, np.int64)
    extra[split] = counts[query[split]] - (end - start)[split]
    ex_off = np.zeros(R + 1, np.int64)
    ex_off[1:] = np.cumsum(xlen + extra)
    ex_rows = np.zeros(int(ex_off[-1]), np.int64)
    if xlen.sum():
        seg = np.repeat(np.arange(R), xlen)
        within = np.arange(int(xlen.sum()), dtype=np.int64) - np.repeat(np.cumsum(xlen) - xlen, xlen)
        ex_rows[ex_off[seg] + within] = np.asarray(excl_rows, np.int64)[np.asarray(excl_offsets, np.int64)[query[seg]] + within]
    for p in split:
        q = query[p]
        ex_rows[ex_off[p] + xlen[p]:ex_off[p + 1]] = np.concatenate([tr[to[q]:start[p]], tr[end[p]:to[q + 1]]])
    return query, offsets, ex_rows, ex_off


def pool_ranks(users, news, tgt_rows, tgt_offsets, excl_rows=None, excl_offsets=None):
    """Ranks of target news among the whole pool under nr_topk_dot's scores (nr_pool_ranks): query q (users (Q, D) fp32)
    has targets tgt_rows[tgt_offsets[q] .. tgt_offsets[q + 1]) of news (n, D) fp32 and optional exclusions in CSR form.
    rank(q, t) is t's 0-based position in the order top_k_scores returns for q over the pool without q's exclusions and
    its other targets: higher score first, equal scores by lower row.  Returns (rank (n_targets,) int64, score
    (n_targets,) fp32 = s(q, t)) in target order, on the caller's stream.  Queries with more than 32 targets run as several
    kernel rows (target_parts).  Raises NewsrecError on bad arguments (before any launch), IndexError on a target or
    exclusion row outside [0, n) and ValueError on a non-finite score (the device flags are read once: one
    synchronisation)."""
    import numpy as np
    lib = load_library()
    if users.dim() != 2 or news.dim() != 2 or users.shape[1] != news.shape[1]:
        raise NewsrecError(f"pool_ranks: users {tuple(users.shape)} and news {tuple(news.shape)} must be (Q, D) and (n, D)")
    if (excl_rows is None) != (excl_offsets is None):
        raise NewsrecError("pool_ranks: excl_rows and excl_offsets go together")
    to = torch.as_tensor(tgt_offsets).cpu().long().numpy()
    Q, D = users.shape
    n = news.shape[0]
    if to.ndim != 1 or len(to) != Q + 1 or to[0] != 0 or (np.diff(to) < 0).any() or to[-1] != len(tgt_rows):
        raise NewsrecError("pool_ranks: tgt_offsets must be (Q + 1,), start at 0, not decrease and end at len(tgt_rows)")
    eo = er = None
    if excl_offsets is not None:
        eo = torch.as_tensor(excl_offsets).cpu().long().numpy()
        er = torch.as_tensor(excl_rows).cpu().long().numpy()
        if eo.ndim != 1 or len(eo) != Q + 1 or er.ndim != 1 or (np.diff(eo) < 0).any() or eo[0] < 0 or eo[-1] > len(er):
            raise NewsrecError("pool_ranks: excl_offsets must be (Q + 1,) non-decreasing offsets into the 1-D excl_rows")
    dev = require_cuda()
    n_t = int(to[-1])
    if int(lib.nr_pool_ranks_workspace(max(Q, 0), max(n, 1), D)) < 0:
        check(-1, "nr_pool_ranks_workspace")
    if n_t == 0:
        return torch.zeros(0, dtype=torch.int64, device=dev), torch.zeros(0, dtype=torch.float32, device=dev)
    if n == 0:
        raise IndexError("pool_ranks: a target row is outside the news pool (the pool is empty)")
    tr = torch.as_tensor(tgt_rows).cpu().long().numpy()
    query, offsets, xr, xo = target_parts(tr, to, er, eo)
    R = len(query)
    users = users.to(dev).float()
    same = R == Q and bool((query == np.arange(Q)).all())
    rows = users.contiguous() if same else users.index_select(0, torch.from_numpy(query).to(dev)).contiguous()
    news = news.to(dev).float().contiguous()
    ws_bytes = int(lib.nr_pool_ranks_workspace(R, n, D))
    if ws_bytes < 0:
        check(-1, "nr_pool_ranks_workspace")
    d_to = torch.from_numpy(offsets).to(dev)
    d_tr = torch.from_numpy(tr).to(dev)
    d_xo = d_xr = None
    if eo is not None or len(xr):
        d_xo = torch.from_numpy(xo).to(dev)
        d_xr = torch.from_numpy(xr if len(xr) else np.zeros(1, np.int64)).to(dev)  # a valid address for an empty set
    rank = torch.empty(n_t, dtype=torch.int64, device=dev)
    score = torch.empty(n_t, dtype=torch.float32, device=dev)
    flags = torch.zeros(3, dtype=torch.int32, device=dev)
    workspace = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    check(lib.nr_pool_ranks(_p(rows), R, D, _p(news), n, D, D, _p(d_to), _p(d_tr), _p(d_xo), _p(d_xr), _p(rank), _p(score),
                            _p(flags[0:1]), _p(flags[1:2]), _p(flags[2:3]), _p(workspace), ws_bytes, _stream()), "nr_pool_ranks")
    bad_row, bad_score, too_many = (int(x) for x in flags.tolist())
    if bad_row:
        raise IndexError("pool_ranks: a target or exclusion row is outside the news pool")
    if bad_score:
        raise ValueError("pool_ranks: a score is not finite; the ranks are undefined")
    if too_many:
        raise NewsrecError("pool_ranks: a kernel row got more than 32 targets")
    return rank, score
