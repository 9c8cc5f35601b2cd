"""Host-side checks of the LSTUR GRU (no device needed).

* The fp64 step functions and backward chain that tests/test_gpu_gru.py holds the kernels to (gpu_checks.gru_proj, gru_step,
  gru_bwd_chain) are themselves checked against torch.autograd through the oracle's packed-sequence GRU: exactly, and under
  the bf16 storage contract with its roundings inserted (plain bf16 x, and x as a hi/lo pair), with lengths 0, 1, S - 1 and S
  in no order.  A chain that drops the r factor of dgh_n misses by far: a wrong reference cannot pass a wrong kernel.
* nr_gru_fwd / _bwd reject a shape outside their rules, and a short backward workspace, with -1 and a message that names the
  cause, before anything is launched.
* The workspace layout the GPU test reads the backward's intermediates through is the library's: the Python restatement of
  gru.cu's GruBwdWorkspace gives nr_gru_bwd_workspace over a grid of shapes."""
import ctypes

import pytest
import torch

import gpu_checks as G
import newsrec_oracle as O


def _lib():
    import os

    import newsrec_b200
    if not os.path.exists(newsrec_b200.LIB_PATH):
        pytest.skip("library not built (python __graft_entry__.py build)")
    return newsrec_b200.load_library()


# ------------------------------------------------------------------------------------------------
def _case(seed, B=5, S=6, D=12, Hd=8):
    bf = lambda t: t.double().to(torch.bfloat16).double()  # the kernels' weights are bf16 operands
    a = Hd ** -0.5
    p = {"g.weight_ih_l0": bf(O.det_uniform((3 * Hd, D), seed, -a, a)), "g.weight_hh_l0": bf(O.det_uniform((3 * Hd, Hd), seed + 1, -a, a)),
         "g.bias_ih_l0": O.det_uniform((3 * Hd,), seed + 2, -a, a).double(), "g.bias_hh_l0": O.det_uniform((3 * Hd,), seed + 3, -a, a).double()}
    x = O.det_uniform((B, S, D), seed + 4).double()
    h0 = O.det_uniform((B, Hd), seed + 5, -0.5, 0.5).double()
    lens = torch.tensor([S - 1, 0, S, 1, 3])[:B]  # unsorted, 0 is clamped to 1
    return p, x, h0, lens, O.det_uniform((B, Hd), seed + 6).double()


def _chain_inputs(p, x, h0, L, contract):
    """What the kernels would store: gi from the operand rows of x (bf16 under the plain contract; the fp64 values where x enters
    as a hi/lo pair or exactly), then the recurrence with gh[t] from h as the recurrent GEMM reads it."""
    rnd = (lambda t: t.to(torch.bfloat16).double()) if contract != "exact" else (lambda t: t)
    xin = rnd(x) if contract == "bf16" else x
    B, S, D = x.shape
    Hd = h0.shape[1]
    W1, W2, b1, b2 = p["g.weight_ih_l0"], p["g.weight_hh_l0"], p["g.bias_ih_l0"], p["g.bias_hh_l0"]
    gi = G.gru_proj(xin.transpose(0, 1).reshape(S * B, D), W1, b1)[0].view(S, B, 3 * Hd)
    hs, gh, hops = [h0], [], []
    for t in range(S):
        hops.append(rnd(hs[t]))
        gh.append(G.gru_proj(hops[t], W2, b2)[0])
        hs.append(G.gru_step(gi[t], gh[t], hs[t], t < L))
    one = torch.ones(S, B, 1, dtype=torch.float64)
    x_ext = torch.cat([xin.transpose(0, 1), one], 2)
    h_ext = torch.cat([torch.stack(hops), one], 2)
    return gi, torch.stack(gh), torch.stack(hs), x_ext, h_ext


@pytest.mark.parametrize("contract", ["exact", "bf16", "bf16_fused"])
def test_backward_chain_matches_autograd_through_the_oracle(contract):
    c = {"exact": O.EXACT, "bf16": O.BF16, "bf16_fused": O.BF16_FUSED}[contract]
    p, x, h0, lens, dout = _case(200 + len(contract))
    L = lens.clamp(min=1)
    p = {k: v.clone().requires_grad_(True) for k, v in p.items()}
    xl, hl = x.clone().requires_grad_(True), h0.clone().requires_grad_(True)
    out = O.gru_last_hidden(xl, L, hl, p, "g", c)
    out.backward(dout)
    with torch.no_grad():
        pd = {k: v.detach() for k, v in p.items()}
        gi, gh, hs, x_ext, h_ext = _chain_inputs(pd, x, h0, L, contract)
        ch = G.gru_bwd_chain(gi, gh, hs, L, pd["g.weight_ih_l0"], pd["g.weight_hh_l0"], x_ext, h_ext, dout, contract=contract != "exact")
        # and with the chain's own dgh handed back as the "stored" one: the same numbers
        ch2 = G.gru_bwd_chain(gi, gh, hs, L, pd["g.weight_ih_l0"], pd["g.weight_hh_l0"], x_ext, h_ext, dout, contract=contract != "exact",
                              dgh_stored=ch["dgh"])
    rel = lambda a, b: float((a - b).norm() / b.norm())
    assert rel(hs[-1], out.detach()) < 1e-12
    B, S, D = x.shape
    assert rel(ch["dx"].transpose(0, 1), xl.grad) < 1e-12
    assert rel(ch["dh0"], hl.grad) < 1e-12
    assert rel(ch["dWih"][:, :D], p["g.weight_ih_l0"].grad) < 1e-12 and rel(ch["dWih"][:, D], p["g.bias_ih_l0"].grad) < 1e-12
    Hd = h0.shape[1]
    assert rel(ch["dWhh"][:, :Hd], p["g.weight_hh_l0"].grad) < 1e-12 and rel(ch["dWhh"][:, Hd], p["g.bias_hh_l0"].grad) < 1e-12
    assert torch.equal(ch["dh0"], ch2["dh0"]) and torch.equal(ch["dgi"], ch2["dgi"])
    # frozen steps (t >= max(len, 1)) carry no gate gradient, and dh arrives at the last active step as dout itself
    act = torch.arange(S).view(S, 1) < L.view(1, B)
    assert bool((ch["dgi"][~act] == 0).all()) and bool((ch["dgh"][~act] == 0).all())
    for b in range(B):
        assert torch.equal(ch["dh"][int(L[b]) - 1, b], dout[b])
    if contract != "exact":  # the contract's roundings are in the chain: every stored gradient is a bf16 value
        assert torch.equal(ch["dgi"], ch["dgi"].to(torch.bfloat16).double()) and torch.equal(ch["dgh"], ch["dgh"].to(torch.bfloat16).double())
    # gru_reference (the end-to-end reference of the GPU test) is the same chain: every output and gradient as autograd's
    ref = G.gru_reference(x, h0, L, *(pd[k] for k in ("g.weight_ih_l0", "g.weight_hh_l0", "g.bias_ih_l0", "g.bias_hh_l0")), dout,
                          contract={"exact": None, "bf16": "bf16", "bf16_fused": "hilo"}[contract])
    assert rel(ref["out"], out.detach()) < 1e-12 and rel(ref["dx"], xl.grad) < 1e-12 and rel(ref["dh0"], hl.grad) < 1e-12
    assert rel(ref["dWhh"][:, :Hd], p["g.weight_hh_l0"].grad) < 1e-12 and rel(ref["dWih"][:, D], p["g.bias_ih_l0"].grad) < 1e-12
    if contract == "bf16_fused":  # the weight gradient reads the bf16 x rows the kernels keep, not the hi/lo pair
        want = ch["dgi"].reshape(-1, 3 * Hd).t() @ x.transpose(0, 1).to(torch.bfloat16).double().reshape(-1, D)
        assert rel(ref["dWih"][:, :D], want) < 1e-12 and rel(ref["dWih"][:, :D], p["g.weight_ih_l0"].grad) > 1e-4
    else:
        assert rel(ref["dWih"][:, :D], p["g.weight_ih_l0"].grad) < 1e-12


def test_chain_without_r_in_dgh_n_fails():
    """dgh_n = dpn (the r factor dropped) gives a W_hh gradient far from autograd's: the chain sees that factor."""
    p, x, h0, lens, dout = _case(230)
    L = lens.clamp(min=1)
    pl = {k: v.clone().requires_grad_(True) for k, v in p.items()}
    O.gru_last_hidden(x, L, h0, pl, "g", O.EXACT).backward(dout)
    gi, gh, hs, x_ext, h_ext = _chain_inputs(p, x, h0, L, "exact")
    Hd = h0.shape[1]
    g = G.gru_gates(gi, gh, Hd)
    ch = G.gru_bwd_chain(gi, gh, hs, L, p["g.weight_ih_l0"], p["g.weight_hh_l0"], x_ext, h_ext, dout)
    wrong = ch["dgh"].clone()
    wrong[..., 2 * Hd:] = torch.where(g["r"] > 0, ch["dgh"][..., 2 * Hd:] / g["r"], 0.0)
    dWhh_wrong = wrong.reshape(-1, 3 * Hd).t() @ h_ext.reshape(-1, Hd + 1)
    rel = lambda a, b: float((a - b).norm() / b.norm())
    assert rel(ch["dWhh"][:, :Hd], pl["g.weight_hh_l0"].grad) < 1e-12
    assert rel(dWhh_wrong[:, :Hd], pl["g.weight_hh_l0"].grad) > 1e-2


def test_step_with_b_hn_outside_r_differs():
    """The cuDNN-style candidate tanh(gi_n + r (gh_n - b_hn) + b_hn) is not torch's: the step function is torch's."""
    p, x, h0, lens, _ = _case(240)
    L = lens.clamp(min=1)
    gi, gh, hs, _, _ = _chain_inputs(p, x, h0, L, "exact")
    Hd = h0.shape[1]
    assert float((hs[-1] - O.gru_last_hidden(x, L, h0, p, "g", O.EXACT)).abs().max()) < 1e-14
    g = G.gru_gates(gi[0], gh[0], Hd)
    bhn = p["g.bias_hh_l0"][2 * Hd:]
    n_cudnn = torch.tanh(gi[0, :, 2 * Hd:] + g["r"] * (gh[0, :, 2 * Hd:] - bhn) + bhn)
    assert float((n_cudnn - g["n"]).abs().max()) > 1e-3


# ------------------------------------------------------------------------------------------------
def _fwd(lib, B, S, D, Hd, **ptrs):
    import newsrec_b200 as nb
    a = nb.GruFwdArgs()
    a.B, a.S, a.D, a.Hd = B, S, D, Hd
    for k, v in ptrs.items():
        setattr(a, k, v)
    return lib.nr_gru_fwd(ctypes.byref(a), None)


def _bwd(lib, B, S, D, Hd, **fields):
    import newsrec_b200 as nb
    a = nb.GruBwdArgs()
    a.B, a.S, a.D, a.Hd = B, S, D, Hd
    for k, v in fields.items():
        setattr(a, k, v)
    return lib.nr_gru_bwd(ctypes.byref(a), None)


@pytest.mark.parametrize("which", ["fwd", "bwd"])
@pytest.mark.parametrize("shape,cause", [
    ((4, 5, 64, 33), "Hd=33"),     # odd hidden size
    ((4, 5, 64, 6), "Hd=6"),       # below 8
    ((4, 5, 62, 64), "D=62"),      # D % 4 != 0
    ((4, 0, 64, 64), "S=0"),       # no step
    ((-1, 5, 64, 64), "B=-1"),     # negative batch
])
def test_bad_shapes_are_rejected_before_launch(which, shape, cause):
    lib = _lib()
    n0 = lib.nr_launch_count()
    rc = (_fwd if which == "fwd" else _bwd)(lib, *shape)
    msg = lib.nr_last_error().decode()
    assert rc == -1 and cause in msg and f"nr_gru_{which}" in msg and lib.nr_launch_count() == n0, (rc, msg)


def test_short_workspace_is_rejected_before_launch():
    lib = _lib()
    B, S, D, Hd = 4, 5, 64, 64
    need = int(lib.nr_gru_bwd_workspace(B, S, D, Hd))
    fake = 1 << 20  # never dereferenced: the workspace check comes before any launch
    n0 = lib.nr_launch_count()
    rc = _bwd(lib, B, S, D, Hd, **{k: fake for k in ("len", "wihT_bf16", "whhT_bf16", "xb", "gi", "gh", "hs", "hb", "dout", "dWih_ext",
                                                     "dWhh_ext", "dx", "dh0", "workspace")}, workspace_bytes=need - 1)
    msg = lib.nr_last_error().decode()
    assert rc == -1 and "workspace too small" in msg and str(need) in msg and lib.nr_launch_count() == n0, (rc, msg)


@pytest.mark.parametrize("B", [0, 1, 37, 129, 512, 2000])
@pytest.mark.parametrize("S,Hd", [(1, 8), (50, 450), (50, 900), (7, 1028), (200, 96)])
def test_workspace_layout_matches_the_library(B, S, Hd):
    lib = _lib()
    lay, total = G.gru_bwd_workspace_layout(B, S, Hd)
    assert total == int(lib.nr_gru_bwd_workspace(B, S, 300, Hd)), (B, S, Hd, lay)
    assert all(v % 256 == 0 for v in lay.values()) and lay["dgi"] == 0 <= lay["dgh"] <= lay["dh_direct"] <= lay["dh_rec"] < total
    assert B == 0 or lay["dgh"] > 0
