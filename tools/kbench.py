"""Micro-benchmarks of single C-ABI operators at BASELINE sizes (CUDA events on the launching stream, L2 flushed
between repetitions by a 256 MB memset).  A tuning tool; bench.py is the contract benchmark.

    python tools/kbench.py [op ...]      ops: mhsa_fwd mhsa_fwd_drop mhsa_bwd qkv pool tn900 tn200 gather dx_fp32 lin:N:K
                                         scatter scatter_live

scatter / scatter_live: the embedding-gradient scatter at the NRMS shape (M = 563,200, N = 300, K = 912) through
nr_element_encoder_bwd, with ids drawn like bench.synth_slots (histories of U{1..50} news left-padded with all-zero news,
titles of U{5..20} tokens right-padded) or all valid; the library's own launch timers give the scatter's kernels apart from
the ReLU backward and weight gradient around them.
"""
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "news-recommendation_b200", "src"))
import torch  # noqa: E402

from newsrec_b200 import check, load_library  # noqa: E402
from newsrec_b200.ops import _p, _stream, ru8, ru16  # noqa: E402

lib = load_library()
dev = torch.device("cuda", 0)
n_seq, T, d, heads, q = 512 * 55, 20, 300, 15, 200
n_tok = n_seq * T
sec = ru8(d)  # Q | K | V sections at columns 0, sec, 2*sec (ops.qkv_pitches)
ldx, ld3, ldq = ru8(d + 1), ru16(3 * sec), ru16(q)
bf = lambda *s: (torch.randn(*s, device=dev) * 0.5).to(torch.bfloat16)
X, QKV, Cx, dC, dQKV = bf(n_tok, ldx), bf(n_tok, ld3), bf(n_tok, ldx), bf(n_tok, ldx), bf(n_tok, ld3)
Wqkv, WqkvT, Wa, WaT = bf(3 * d, ldx), bf(d, ld3), bf(q, ldx), bf(d, ldq)
dpre = bf(n_tok, ldq)
bias3, ba, qv = torch.randn(3 * d, device=dev), torch.randn(q, device=dev), torch.randn(q, device=dev) * 0.1
w = torch.rand(n_tok, device=dev)
out = torch.empty(n_seq, d, device=dev)
dout = torch.randn(n_seq, d, device=dev)
ids = torch.randint(1, 70976, (n_tok,), device=dev)
demb = torch.zeros(70976, d, device=dev)
table = bf(70976, ldx)
dW = torch.zeros(3 * d, ldx, device=dev)
flag = torch.zeros(1, dtype=torch.int32, device=dev)
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
st = _stream()

OPS = {
    "mhsa_fwd": lambda: lib.nr_mhsa_core_fwd(_p(QKV), ld3, sec, n_seq, T, heads, d // heads, _p(Cx), ldx, 0.0, 0, st),
    "mhsa_fwd_drop": lambda: lib.nr_mhsa_core_fwd(_p(QKV), ld3, sec, n_seq, T, heads, d // heads, _p(Cx), ldx, 0.2, 1234, st),
    "mhsa_bwd": lambda: lib.nr_mhsa_core_bwd(_p(QKV), ld3, sec, _p(dC), ldx, n_seq, T, heads, d // heads, _p(dQKV), ld3, st),
    "qkv": lambda: lib.nr_linear(_p(X), n_tok, ldx, _p(Wqkv), 3 * d, ldx, d, 1, 0, 128, _p(bias3), 0, _p(QKV), ld3, 1, st),
    "pool": lambda: lib.nr_additive_attention_fwd(_p(Cx), n_seq, T, d, ldx, _p(Wa), q, ldx, _p(ba), _p(qv), _p(out), d, _p(w), st),
    "tn900": lambda: lib.nr_gemm_tn(_p(dQKV), n_tok, 3 * d, ld3, _p(X), n_tok, d + 1, ldx, 0, d + 1, 0, _p(dW), ldx, st),
    "tn200": lambda: lib.nr_gemm_tn(_p(dpre), n_tok, q, ldq, _p(Cx), n_tok, d + 1, ldx, 0, d + 1, 0, _p(dW), ldx, st),
    "gather": lambda: lib.nr_gather_rows(_p(ids), n_tok, T, _p(table), 70976, d, ldx, _p(X), 0, 0.2, 99, _p(flag), st),
    "dx_fp32": lambda: lib.nr_linear(_p(dQKV), n_tok, ld3, _p(WqkvT), d, ld3, 3 * d, 1, 0, 128, None, 0, _p(demb_big), d, 0, st),
}
demb_big = None
names = sys.argv[1:] or ["mhsa_fwd", "mhsa_fwd_drop", "mhsa_bwd", "qkv", "pool", "tn900", "tn200", "gather"]
if "dx_fp32" in names:
    demb_big = torch.empty(n_tok, d, device=dev)
def synth_title_ids(B=512, H=50, C=5, T=20, V=70976, seed=0):
    """news-level token ids in the encoder's order: the B x H browsed news, then the B x C candidates"""
    g = torch.Generator().manual_seed(seed)
    hl = torch.randint(1, H + 1, (B,), generator=g)
    ids = torch.randint(1, V, (B, H + C, T), generator=g) * (torch.arange(T) < torch.randint(5, T + 1, (B, H + C, 1), generator=g))
    ids[:, :H] *= (torch.arange(H).view(1, -1, 1) >= H - hl.view(-1, 1, 1))
    return torch.cat([ids[:, :H].reshape(-1), ids[:, H:].reshape(-1)]).to(dev)


def scatter_op(all_live):
    """nr_element_encoder_bwd with E = d, F = 3 * sec: its scatter is gemm_scatter_emb at the NRMS shape"""
    E, F, V = d, 3 * sec, 70976
    lde, ldf = ru8(E + 1), ru8(F + 1)
    sids = torch.randint(1, V, (n_tok,), device=dev) if all_live else synth_title_ids(V=V)
    dout, out = torch.randn(n_tok, F, device=dev), torch.ones(n_tok, F, device=dev)
    dY, Eb, WT = torch.empty(n_tok, ldf, device=dev, dtype=torch.bfloat16), bf(n_tok, lde), bf(E, ldf)
    dWe, dt = torch.zeros(F, lde, device=dev), torch.zeros(V, E, device=dev)
    print(f"scatter ids: {float(((sids >= 1) & (sids < V)).float().mean()):.3f} of the rows valid", flush=True)
    return lambda: lib.nr_element_encoder_bwd(_p(sids), n_tok, _p(dout), _p(out), F, _p(dY), ldf, _p(Eb), E, lde, _p(WT), _p(dWe),
                                              _p(dt), V, st)


def lin_op(spec):
    """lin:N:K[:bf16out] -> nr_linear at M = n_tok with fresh operands"""
    parts = spec.split(":")
    N, K = int(parts[1]), int(parts[2])
    lda, ldo = ru8(K + 1), ru16(N)
    A, W, O = bf(n_tok, lda), bf(N, lda), torch.empty(n_tok, ldo, device=dev, dtype=torch.bfloat16)
    b = torch.randn(N, device=dev)
    return lambda: lib.nr_linear(_p(A), n_tok, lda, _p(W), N, lda, K, 1, 0, 128, _p(b), 0, _p(O), ldo, 1, st)


for name in names:
    if name in ("scatter", "scatter_live"):
        fn = scatter_op(name == "scatter_live")
        for _ in range(2):
            check(fn(), name)
        lib.nr_profile_enable(1)
        for _ in range(5):
            flush.zero_()
            check(fn(), name)
        torch.cuda.synchronize()
        lib.nr_profile_enable(0)
        buf = C.create_string_buffer(1 << 16)
        assert lib.nr_profile_report(buf, len(buf)) >= 0
        for key, (count, ms) in json.loads(buf.value.decode()).items():
            if "scatter" in key:
                print(f"{name:15s} {key:50s} {ms / count:.4f} ms per call ({count} calls)", flush=True)
        continue
    fn = lin_op(name) if name.startswith("lin:") else OPS[name]
    for _ in range(2):
        check(fn(), name)
    ts = []
    for _ in range(5):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        check(fn(), name)
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    print(f"{name:15s} min {min(ts):.4f} ms  med {sorted(ts)[2]:.4f} ms", flush=True)
