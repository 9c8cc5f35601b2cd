"""Host-side checks of the self-attention encoder (no device needed).

* nr_mhsa_encoder_fwd / _bwd reject a head size outside the attention kernels' range 2 <= d_k <= 32 with -1 before any
  launch (include/newsrec_b200.h): the check runs before any pointer or device is touched.
* The fp64 backward chain that tests/test_gpu_mhsa_encoder.py holds the kernels to (gpu_checks.mhsa_pool_bwd_chain) is
  itself checked against torch.autograd through the oracle's self-attention and additive pooling, exactly and under the
  bf16 storage contract, with and without the dropout masks: a wrong reference cannot pass a wrong kernel."""
import ctypes

import pytest
import torch

import gpu_checks as G
import newsrec_oracle as O


def _lib():
    import newsrec_b200
    import os
    if not os.path.exists(newsrec_b200.LIB_PATH):
        pytest.skip("library not built (python __graft_entry__.py build)")
    return newsrec_b200.load_library()


def _call(which, heads, d=300, T=20, q=200):
    import newsrec_b200 as nb
    from newsrec_b200.ops import qkv_pitches, ru8, ru16
    lib = _lib()
    a = nb.MhsaEncoderFwdArgs() if which == "fwd" else nb.MhsaEncoderBwdArgs()
    a.n_seq, a.T, a.d, a.heads, a.q, a.ldx, a.ld3 = 8, T, d, heads, q, ru8(d + 1), qkv_pitches(d)[1]
    if which == "bwd":
        a.ldq = ru16(q)
    n0 = lib.nr_launch_count()
    fn = lib.nr_mhsa_encoder_fwd if which == "fwd" else lib.nr_mhsa_encoder_bwd
    rc = fn(ctypes.byref(a), None)
    return rc, lib.nr_last_error().decode(), lib.nr_launch_count() - n0


@pytest.mark.parametrize("which", ["fwd", "bwd"])
@pytest.mark.parametrize("heads,dk", [(5, 60), (300, 1)])
def test_head_size_outside_the_kernels_is_rejected_before_launch(which, heads, dk):
    rc, msg, launched = _call(which, heads)
    assert rc == -1 and f"d_k={dk}" in msg and launched == 0, (rc, msg, launched)


@pytest.mark.parametrize("which", ["fwd", "bwd"])
@pytest.mark.parametrize("heads", [150, 10])
def test_head_sizes_at_the_ends_pass_the_shape_check(which, heads):
    """d_k = 2 and d_k = 30 pass the shape check: with null operands the call fails on the pointers instead, still before any
    launch."""
    rc, msg, launched = _call(which, heads)
    assert rc == -1 and not msg.startswith("mhsa encoder:") and launched == 0, (rc, msg, launched)


# ------------------------------------------------------------------------------------------------
def _params(d, q, seed):
    r = lambda shape, s, a: O.det_uniform(shape, s, -a, a).double()
    bf = lambda t: t.to(torch.bfloat16).double()  # the kernels' operands are bf16 values
    p = {}
    for i, n in enumerate("QKV"):
        p[f"m.W_{n}.weight"] = bf(r((d, d), seed + i, 3.0 / d ** 0.5))
        p[f"m.W_{n}.bias"] = r((d,), seed + 3 + i, 0.1)
    p["a.linear.weight"] = bf(r((q, d), seed + 6, (3.0 / d) ** 0.5))
    p["a.linear.bias"] = r((q,), seed + 7, 0.1)
    p["a.attention_query_vector"] = r((q,), seed + 8, 1.0)
    return {k: v.requires_grad_(True) for k, v in p.items()}


def _mask(shape, seed, p=0.25):
    keep = O.det_uniform(shape, seed, 0.0, 1.0) >= p
    return keep.double() / (1.0 - p)


@pytest.mark.parametrize("contract", [False, True])
@pytest.mark.parametrize("masks", [False, True])
def test_backward_chain_matches_autograd_through_the_oracle(contract, masks):
    n, T, d, heads, q, V = 3, 7, 12, 3, 6, 9
    c = O.BF16 if contract else O.EXACT
    p = _params(d, q, 100 + 2 * contract + masks)
    table = O.det_uniform((V, d), 5).double().to(torch.bfloat16).double().requires_grad_(True)
    ids = O.det_randint((n, T), 6, 0, V)
    ids[0, 0], ids[1, 2] = 0, V - 1
    mx = _mask((n, T, d), 7) if masks else torch.ones(n, T, d, dtype=torch.float64)
    cm = _mask((n, T, d), 8) if masks else None
    # forward with autograd: masked gather, the oracle's projection / attention / pooling; the context mask is applied before
    # the one bf16 store of the context gradient, as the pooling-backward kernel does
    x = table[ids] * mx
    if cm is None:
        ctx = O.multihead_self_attention(x, p, "m", heads, c)
    else:
        proj = lambda k: c.act(torch.nn.functional.linear(x, c.operand(p[f"m.W_{k}.weight"])) + p[f"m.W_{k}.bias"])
        sp = lambda t: t.view(n, T, heads, d // heads).transpose(1, 2)
        a = O.scaled_dot_product_attention(sp(proj("Q")), sp(proj("K")), sp(proj("V")), c)
        ctx = c.grad(a.transpose(1, 2).reshape(n, T, d)) * cm
    out = O.additive_attention(ctx, p, "a", c)
    dout = O.det_uniform((n, d), 9).double()
    out.backward(dout)
    # the chain, from the forward values the kernels would have stored
    with torch.no_grad():
        X = x.detach()
        W3 = torch.stack([p[f"m.W_{k}.weight"] for k in "QKV"]).detach()
        b3 = torch.stack([p[f"m.W_{k}.bias"] for k in "QKV"]).detach()
        st = (lambda t: t.to(torch.bfloat16).double()) if contract else (lambda t: t)
        Q, K, Vv = [st(X @ W3[i].t() + b3[i]) for i in range(3)]
        Cc = ctx.detach()
        Wa, ba, qv = (p[k].detach() for k in ("a.linear.weight", "a.linear.bias", "a.attention_query_vector"))
        w = torch.softmax((torch.tanh(Cc @ Wa.t() + ba) @ qv), dim=1)
        ch = G.mhsa_pool_bwd_chain(X, Q, K, Vv, Cc, w, W3, Wa, ba, qv, dout, heads, ctx_mask=cm, contract=contract)
        demb = torch.zeros(V, d, dtype=torch.float64)
        flat, dX = ids.reshape(-1), (ch["dX"] * mx).reshape(-1, d)
        sc = flat >= 1  # padding_idx 0 gets no gradient
        demb.index_add_(0, flat[sc], dX[sc])
    rel = lambda a, b: float((a - b).norm() / b.norm())
    assert rel(ch["dqv"], p["a.attention_query_vector"].grad) < 1e-12
    assert rel(ch["dWa"][:, :d], p["a.linear.weight"].grad) < 1e-12 and rel(ch["dWa"][:, d], p["a.linear.bias"].grad) < 1e-12
    for i, k in enumerate("QKV"):
        assert rel(ch["dW3"][i, :, :d], p[f"m.W_{k}.weight"].grad) < 1e-12, k
        if k != "K":  # d(b_K) is analytically zero (softmax shift invariance): rounding noise on both sides
            assert rel(ch["dW3"][i, :, d], p[f"m.W_{k}.bias"].grad) < 1e-12, k
    tg = table.grad.clone()
    tg[0] = 0.0  # F.embedding in this graph has no padding_idx; the kernels never write row 0
    assert rel(demb, tg) < 1e-12
    # and the chain is sensitive to what it is given: dropping the context mask changes the weight gradients
    if masks:
        wrong = G.mhsa_pool_bwd_chain(X, Q, K, Vv, Cc, w, W3, Wa, ba, qv, dout, heads, ctx_mask=None, contract=contract)
        assert rel(wrong["dW3"][:, :, :d], torch.stack([p[f"m.W_{k}.weight"].grad for k in "QKV"])) > 1e-2
