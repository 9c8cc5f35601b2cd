"""bench.py -- impressions/sec, forward+backward, on MIND-shaped synthetic batches (BASELINE.json).

    python bench.py --gpus 1 --steps 20 --warmup 5                       # NRMS, BASELINE.json configs[1] (and [4] at N=8)
    python bench.py --model NAML|LSTUR|TANR                              # configs[2], configs[3] (+ TANR)
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P \
        bench.py --gpus N --steps K --warmup W
    python bench.py --impl reference --steps 3 --warmup 1                # the reference's CPU path (oracle port), same batch

One "step" = zero_grad -> forward -> CrossEntropy(label 0) -> backward over one batch of B=512 impressions per GPU
(1+K=5 candidates + 50 browsed titles of 20 tokens each = 55 news encodes + 1 user encode + 5 scores), plus -- for N>1 --
the one NCCL gradient all-reduce.  The optimizer step is excluded: the metric is forward+backward (BASELINE.md section 3).
Prints ONE JSON line on rank 0.

  value    device-resident inputs (slot lists already in HBM)
  e2e      the reference's own call, `model(candidate_news, clicked_news)` with the CPU slot lists a DataLoader yields
           (src/train.py:202): host stacking into pinned memory + one H2D copy + device re-ordering inside forward, and a
           device->host read of the loss every step -- what the unmodified train.py does with the drop-in
  e2e_prefetch   (NRMS) the same with the NEXT batch staged on a copy stream by NRMS.prefetch (an API the reference lacks)
"""
from __future__ import annotations

import argparse
import importlib
import json
import os
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "news-recommendation_b200", "src"))

import torch  # noqa: E402

V_WORDS, T_TITLE, T_ABS, H_HIST, K_NEG, D_MODEL, HEADS, Q_DIM = 70976, 20, 50, 50, 4, 300, 15, 200
N_CAT, N_USERS = 275, 50001
C_CAND = 1 + K_NEG
N_NEWS = C_CAND + H_HIST


def flop_fwd_per_impression(model, F):
    """Algorithmic forward FLOPs per impression (SURVEY.md 8d; padding to MMA shapes is NOT counted); x3 for fwd+bwd."""
    N, T, Ta, d, q, H, C = N_NEWS, T_TITLE, T_ABS, D_MODEL, Q_DIM, H_HIST, C_CAND
    if model == "NRMS":
        dk = d // HEADS
        return (N * T * 6 * d * d + N * HEADS * 4 * T * T * dk + N * T * 2 * d * q + N * T * (2 * q + 2 * d)
                + H * 6 * d * d + HEADS * 4 * H * H * dk + H * 2 * d * q + C * 2 * d)
    conv = lambda L: N * L * 2 * 3 * d * F
    pool = lambda L: N * L * (2 * F * q + 2 * q + 2 * F)
    if model == "NAML":
        return conv(T + Ta) + pool(T + Ta) + N * 2 * 2 * 100 * F + N * 4 * 2 * F * q + H * 2 * F * q
    if model == "TANR":
        return conv(T) + pool(T) + H * 2 * F * q + N * 2 * F * N_CAT
    D = 3 * F  # LSTUR: GRU over the full history length (the synthetic lengths average H/2; the algorithmic figure is quoted at len = H)
    return conv(T) + pool(T) + H * 2 * (3 * D * D) * 2


def bytes_per_impression(model):
    """Compulsory HBM traffic per impression, fwd+bwd (SURVEY.md 8d): bf16 gather + fp32 embedding-gradient write + ids."""
    tok = N_NEWS * (T_TITLE + (T_ABS if model == "NAML" else 0))
    return tok * D_MODEL * 2 + tok * D_MODEL * 4 + tok * 8


WORKLOADS = {
    "NRMS": "NRMS bf16 fwd+bwd: batch={B}/GPU, title_len=20, history=50, K=4, 15 heads x d_k=20, d=300, V=70976",
    "NAML": "NAML bf16 fwd+bwd: batch={B}/GPU, title(20)+abstract(50)+category+subcategory, CNN filters=400 window=3, history=50, K=4, d=300",
    "LSTUR": "LSTUR(ini) bf16 fwd+bwd: batch={B}/GPU, CNN news encoder F=300 + GRU user encoder over history=50, K=4, d=300",
    "TANR": "TANR bf16 fwd+bwd: batch={B}/GPU, CNN news encoder F=300 + additive user encoder + topic head, history=50, K=4",
}
FIELDS = {"NRMS": ("title",), "NAML": ("category", "subcategory", "title", "abstract"), "LSTUR": ("category", "subcategory", "title"),
          "TANR": ("category", "title")}


def synth_slots(model, B, seed, device="cpu", pin=False):
    """MIND-shaped inputs exactly as default_collate hands them to the model: slot-major lists of dicts of (B, ...) int64.
    Title length U{5..20} / abstract U{10..50} right-padded with 0; history length U{1..50}, LEFT-padded with all-zero news."""
    g = torch.Generator().manual_seed(seed)

    def text(T, lo):
        ids = torch.randint(1, V_WORDS, (B, N_NEWS, T), generator=g)
        ln = torch.randint(lo, T + 1, (B, N_NEWS, 1), generator=g)
        return ids * (torch.arange(T).view(1, 1, -1) < ln)

    hl = torch.randint(1, H_HIST + 1, (B,), generator=g)
    keep = (torch.arange(H_HIST).view(1, -1) >= (H_HIST - hl.view(-1, 1)))  # (B, H)
    data = {}
    for f in FIELDS[model]:
        if f == "title":
            t = text(T_TITLE, 5)
        elif f == "abstract":
            t = text(T_ABS, 10)
        else:
            t = torch.randint(1, N_CAT, (B, N_NEWS), generator=g)
        m = keep.view(B, H_HIST, *([1] * (t.dim() - 2)))
        t[:, C_CAND:] = t[:, C_CAND:] * m
        data[f] = t

    def mk(t):
        t = t.contiguous()
        if device != "cpu":
            return t.to(device)
        return t.pin_memory() if pin else t

    cand = [{f: mk(data[f][:, j]) for f in data} for j in range(C_CAND)]
    clicked = [{f: mk(data[f][:, C_CAND + j]) for f in data} for j in range(H_HIST)]
    extra = ()
    if model == "LSTUR":
        extra = (mk(torch.randint(1, N_USERS, (B,), generator=g)), hl.clone())  # (user ids, clicked_news_length on the host)
    return extra, cand, clicked


class ClockSampler:
    """nvidia-smi clocks / throttle reasons sampled DURING the timed region."""
    Q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, index):
        self.rows, self.proc, self.index = [], None, index

    def __enter__(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-lms", "100",
                                          "-i", str(self.index)], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.thread = threading.Thread(target=self._read, daemon=True)
            self.thread.start()
        except OSError:
            self.proc = None
        return self

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([x.strip() for x in line.split(",")])

    def __exit__(self, *a):
        if self.proc is not None:
            self.proc.terminate()
            try:
                self.proc.wait(timeout=2)
            except subprocess.TimeoutExpired:
                self.proc.kill()

    def summary(self):
        sm, mx, reasons = [], [], set()
        for r in self.rows:
            try:
                sm.append(float(r[0]))
                mx.append(float(r[1]))
            except (ValueError, IndexError):
                continue
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), r[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        if not sm:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": [], "samples": 0}
        return {"sm_mhz": statistics.median(sm), "sm_max_mhz": max(mx), "reasons": sorted(reasons), "samples": len(sm)}


def peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return {"hbm_gbs": d["hbm_gbs"], "bf16_tflops": d["bf16_tflops"], "bf16_tflops_sustained": d.get("bf16_tflops_sustained", d["bf16_tflops"]),
                "source": "measured (MEASURED_PEAKS.json)"}
    # NVIDIA H100 SXM data sheet (700 W): 3.35 TB/s HBM3, 989 dense BF16 TFLOP/s; a data-sheet rate, not a measured one
    return {"hbm_gbs": 3350.0, "bf16_tflops": 989.0, "bf16_tflops_sustained": 989.0, "source": "H100 SXM data sheet"}


def kernel_work(name):
    """Algorithmic FLOPs and the kernel's own (unfused) HBM bytes of ONE launch, from the '<ctx>/<op>[a,b,c]' profile key."""
    op = name.split("/")[1].split("[")[0]
    a, b, c = [int(x) for x in name.split("[")[1].rstrip("]").split(",")]
    if op in ("gemm_store", "gemm_scatter_emb"):          # [M, N, K]
        return 2.0 * a * b * c, 2.0 * a * c + (2.0 * a * b if op == "gemm_store" else 4.0 * a * b)
    if op in ("gemm_additive_pool", "gemm_additive_dpre"):  # [M, q, D]
        return 2.0 * a * b * c + 4.0 * a * b, 2.0 * a * c * (2 if op == "gemm_additive_pool" else 1) + 2.0 * a * b
    if op == "gemm_pool_dinput":                           # [M, D, q]
        return 2.0 * a * b * c, 2.0 * a * c + 2.0 * a * b
    if op == "gemm_tn":                                    # [Kr, Ma, Nb]
        return 2.0 * a * b * c, 2.0 * a * (b + c)
    if op == "mhsa_core_fwd":                              # [n_seq, T, d]
        return 4.0 * a * b * b * c, 2.0 * a * b * c * 4
    if op == "mhsa_core_fwd_hilo":                         # accurate mode: + V low plane in, + context low plane out, 3 P.V products
        return 8.0 * a * b * b * c, 2.0 * a * b * c * 6
    if op == "mhsa_core_bwd":
        return 10.0 * a * b * b * c, 2.0 * a * b * c * 7
    if op == "gather_rows":                                # [n_tok, D, ld]
        return 0.0, 2.0 * a * c * 2
    if op == "pool_dscore":                                # [n_seg, seg_len, D]
        return 2.0 * a * b * c, 2.0 * a * b * c
    return 0.0, 0.0


def usable_cores():
    """Host cores this process may actually use: affinity mask capped by the cgroup CPU quota (os.cpu_count()
    reports the whole machine inside a container; oversubscribing OpenMP threads stalls the CPU arm)."""
    n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    try:
        quota, period = open("/sys/fs/cgroup/cpu.max").read().split()
        if quota != "max":
            n = min(n, max(1, int(int(quota) / int(period))))
    except (OSError, ValueError):
        try:
            q = int(open("/sys/fs/cgroup/cpu/cpu.cfs_quota_us").read())
            per = int(open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read())
            if q > 0:
                n = min(n, max(1, q // per))
        except (OSError, ValueError):
            pass
    return min(n, 64)


def log(msg):
    print(f"[bench] {msg}", file=sys.stderr, flush=True)


def run_reference(model, B, steps, warmup, F):
    """The reference's own CPU path on all usable host threads, same shapes and the SAME batch as the GPU arm.
    NRMS: the oracle port with the reference's per-slot call structure, dropout active (train mode).  The CNN families:
    the oracle's functional restatement (fp32 autograd, eval-mode arithmetic: their dropout masks are not restated)."""
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import newsrec_oracle as O
    cores = usable_cores()
    torch.set_num_threads(cores)
    log(f"reference arm ({model}): {cores} threads, batch {B}, {warmup}+{steps} steps")
    batches = [synth_slots(model, B, 100 + i) for i in range(2)]
    if model == "NRMS":
        net = O.ReferenceStructuredNRMS(V_WORDS, D_MODEL, HEADS, Q_DIM, 0.2, 0)
        net.train()
        one = lambda b: O.reference_cpu_step(net, b[1], b[2])
        kind = "torch CPU, fp32, train mode (dropout on), one encoder call per slot as the reference"
    else:
        shapes = {"NAML": lambda: O.naml_shapes(V_WORDS, N_CAT, Fn=F), "TANR": lambda: O.tanr_shapes(V_WORDS, N_CAT, Fn=F),
                  "LSTUR": lambda: O.lstur_shapes(V_WORDS, N_CAT, N_USERS, Fn=F)}[model]()
        p = {k: v.requires_grad_(True) for k, v in O.tie_shared(O.det_state_dict(shapes, 0)).items()}
        stack = lambda lst, f: torch.stack([x[f] for x in lst], dim=1)

        def one(b):
            extra, cand, clicked = b
            for v in p.values():
                v.grad = None
            cd = {f: stack(cand, f) for f in FIELDS[model]}
            hd = {f: stack(clicked, f) for f in FIELDS[model]}
            if model == "NAML":
                loss = O.click_loss(O.naml_forward(cd, hd, p))
            elif model == "TANR":
                lg, tl = O.tanr_forward(cd, hd, p)
                loss = O.click_loss(lg) + 0.1 * tl
            else:
                loss = O.click_loss(O.lstur_forward(extra[0], extra[1], cd, hd, p, "ini"))
            loss.backward()
        kind = "torch CPU, fp32, functional restatement (eval-mode arithmetic)"
    for i in range(warmup):
        one(batches[i % 2])
    t0 = time.perf_counter()
    for i in range(steps):
        one(batches[i % 2])
    dt = time.perf_counter() - t0
    return B * steps / dt, dt / max(steps, 1) * 1e3, cores, kind


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--model", default="NRMS", choices=["NRMS", "NAML", "LSTUR", "TANR"])
    ap.add_argument("--batch", type=int, default=512, help="impressions per GPU per step (BASELINE.json configs[1])")
    ap.add_argument("--ref-batch", type=int, default=0, help="impressions per CPU step of the reference arm (0 = --batch: same configuration)")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-operand-refresh", action="store_true",
                    help="tuning: keep the bf16 operand shadows across steps (as if the weights never changed)")
    ap.add_argument("--quick", action="store_true", help="tuning: device-resident timing only (prints a short JSON line)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write what the last timed step computed (logits, loss, parameter gradients; "
                         "float32 .npy, large gradients as a fixed seeded row sample) to DIR")
    args = ap.parse_args()
    args.warmup = max(args.warmup, 3) if args.impl == "b200" else max(min(args.warmup, 1), 1)
    model_name = args.model
    F = 400 if model_name == "NAML" else 300  # BASELINE.json configs[2]: CNN filters=400
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    workload = WORKLOADS[model_name].format(B=args.batch)
    ref_batch = args.ref_batch or args.batch

    if args.impl == "reference":
        if rank != 0:
            return
        steps = min(args.steps, 6)  # a bounded sample: one CPU step of 512 impressions takes ~10-15 s on 16 cores
        val, ms, cores, kind = run_reference(model_name, ref_batch, steps, args.warmup, F)
        print(json.dumps({
            "metric": "impressions/sec (fwd+bwd)", "value": val, "unit": "impressions/s", "n_gpus": args.gpus, "steps": steps,
            "warmup": args.warmup, "ms_per_step": ms, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "f32", "data": "synthetic", "impl": "reference",
            "config": {"workload": workload, "global_batch": ref_batch, "reference_step_batch": ref_batch},
            "cpu_baseline": {"value": val, "unit": "impressions/s", "cores": cores, "kind": "port",
                             "sample": f"{steps} steps of {ref_batch} impressions (same shapes, same batch as the GPU arm); {kind}"},
            "e2e": {"value": val, "unit": "impressions/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
            "gpu_launches": 0}))
        return

    import newsrec_b200
    from newsrec_b200 import ddp
    rank, world, local = ddp.init_from_env("nccl")
    assert torch.cuda.is_available(), "bench.py --impl b200 needs a CUDA device (no CPU fallback)"
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    import config as cfgmod
    Model = getattr(importlib.import_module("model." + model_name), model_name)
    over = {"num_filters": F} if model_name == "NAML" else ({"long_short_term_method": "ini"} if model_name == "LSTUR" else {})
    cfg = type("Cfg", (getattr(cfgmod, model_name + "Config"),), over)
    lib = newsrec_b200.load_library()
    torch.manual_seed(0)
    model = Model(cfg).to(dev)
    model.train()  # dropout active exactly as in the reference's training step
    grads = ddp.FlatGradients(model.parameters(), world)
    B = args.batch
    n_rot = 3  # rotate distinct batches; the per-step intermediates (> 1 GB) far exceed the 50 MB L2
    dev_batches = [synth_slots(model_name, B, 1000 * rank + i, device=dev) for i in range(n_rot)]
    host_batches = [synth_slots(model_name, B, 1000 * rank + 50 + i, pin=True) for i in range(n_rot)]
    label = torch.zeros(B, dtype=torch.long, device=dev)
    topic_w = getattr(cfg, "topic_classification_loss_weight", 0.1)

    def loss_of(out):
        if isinstance(out, tuple):  # TANR: (click logits, topic loss), train.py:190,224
            return torch.nn.functional.cross_entropy(out[0], label) + topic_w * out[1]
        return torch.nn.functional.cross_entropy(out, label)

    def fwd(batch):
        extra, cand, clicked = batch
        if model_name == "LSTUR":
            return model(extra[0], extra[1].clone(), cand, clicked)  # the reference mutates clicked_news_length in place
        return model(cand, clicked)

    from newsrec_b200.ops import OperandCache
    caches = [c for c in (getattr(m, "_cache", None) for m in model.modules()) if isinstance(c, OperandCache)]

    last = {}

    def step(batch, read_loss=False):
        grads.zero()
        if not args.no_operand_refresh:
            # no optimizer runs in the timed step, so the parameters' version counters never move and the bf16 operand shadows
            # (embedding table [V][304], packed / transposed weights) would be built once and reused for ever; a real training
            # step rebuilds them after every update -- drop them so that the timed step pays for that refresh
            for c in caches:
                c.invalidate_operands()
        out = fwd(batch)
        loss = loss_of(out)
        loss.backward()
        grads.all_reduce_mean()
        last["out"], last["loss"] = out, loss
        return loss.item() if read_loss else None

    def dump_outputs(d):
        """The arrays a caller of the timed step receives after its last step: the click logits (TANR: and the topic loss), the
        loss and every parameter gradient.  Gradients above 1M elements are sampled: 1024 rows drawn with a fixed seed."""
        import numpy as np
        os.makedirs(d, exist_ok=True)
        torch.cuda.synchronize()
        out = last["out"]
        arrays = {"logits": out[0] if isinstance(out, tuple) else out, "loss": last["loss"].reshape(1)}
        if isinstance(out, tuple):
            arrays["topic_loss"] = out[1].reshape(1)
        g = torch.Generator().manual_seed(1234)
        for name, prm in model.named_parameters():
            if prm.grad is None:
                continue
            gr = prm.grad.detach()
            if gr.numel() > (1 << 20):
                rows = torch.sort(torch.randperm(gr.shape[0], generator=g)[:1024]).values
                np.save(os.path.join(d, f"grad.{name}.rows.npy"), rows.numpy().astype(np.float64))
                gr = gr[rows.to(gr.device)]
            arrays["grad." + name] = gr
        for k, v in arrays.items():
            np.save(os.path.join(d, k + ".npy"), v.detach().float().cpu().numpy())

    def barrier():
        if world > 1:
            torch.distributed.barrier()
        torch.cuda.synchronize()

    def max_ms(e0, e1):
        ms = torch.tensor([e0.elapsed_time(e1)], device=dev)
        if world > 1:
            torch.distributed.all_reduce(ms, op=torch.distributed.ReduceOp.MAX)
        return float(ms.item())

    def timed(batches, read_loss, profile=False):
        for i in range(args.warmup):
            step(batches[i % n_rot], read_loss)
        barrier()
        if profile:  # per-kernel CUDA events cover the TIMED steps only (first launches pay lazy module loading)
            lib.nr_profile_enable(1)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        l0 = newsrec_b200.launch_count()
        e0.record()
        for i in range(args.steps):
            step(batches[i % n_rot], read_loss)
        e1.record()
        barrier()
        return max_ms(e0, e1), newsrec_b200.launch_count() - l0

    def timed_prefetch(batches):
        """NRMS only: every timed step stages the NEXT batch (host stacking + H2D + device re-ordering) on a copy stream
        while this step's kernels run, and reads its own loss back."""
        def run(n):
            cur = model.prefetch(batches[0][1], batches[0][2])
            for i in range(n):
                grads.zero()
                loss = torch.nn.functional.cross_entropy(model(cur), label)
                loss.backward()
                grads.all_reduce_mean()
                if i + 1 < n:
                    nb = batches[(i + 1) % n_rot]
                    cur = model.prefetch(nb[1], nb[2])
                loss.item()
        run(args.warmup)
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        run(args.steps)
        e1.record()
        barrier()
        return max_ms(e0, e1)

    log(f"rank {rank}/{world}: {model_name} + data ready; timing device-resident steps")
    with ClockSampler(local) as clk:
        ms_total, launches = timed(dev_batches, read_loss=False)
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs)
    if args.quick:
        if world > 1:
            torch.distributed.barrier()
            torch.cuda.synchronize()
            torch.distributed.destroy_process_group()
        if rank == 0:
            print(json.dumps({"quick": True, "n_gpus": world, "ms_per_step": ms_total / args.steps,
                              "value": B * world * args.steps / (ms_total / 1e3),
                              "env": {k: os.environ.get(k) for k in ("NEWSREC_COMM_SMS", "NCCL_MAX_NCHANNELS", "NCCL_MIN_NCHANNELS")}}), flush=True)
        return
    log(f"device-resident: {ms_total / args.steps:.3f} ms/step; per-kernel pass")
    timed(dev_batches, read_loss=False, profile=True)  # separate pass: the event pairs around every launch stay out of `value`
    prof = newsrec_b200.profile_report()
    lib.nr_profile_enable(0)
    log("timing end-to-end steps (host slot lists through model(candidate_news, clicked_news), loss read back)")
    ms_e2e, _ = timed(host_batches, read_loss=True)
    log(f"end-to-end (reference API): {ms_e2e / args.steps:.3f} ms/step")
    ms_pref = timed_prefetch(host_batches) if model_name == "NRMS" else None

    log(f"rank {rank}: timed regions done")
    if world > 1:
        torch.distributed.barrier()
        torch.cuda.synchronize()
        torch.distributed.destroy_process_group()
    log(f"rank {rank}: process group closed")
    if rank != 0:
        return
    pk = peaks()
    imp = B * world * args.steps
    value = imp / (ms_total / 1e3)
    e2e = imp / (ms_e2e / 1e3)
    # dominant kernel of the step and its roofline (timed inside a long step -> sustained tensor peak)
    tot_prof = sum(v[1] for v in prof.values())
    dom = max(prof.items(), key=lambda kv: kv[1][1])
    flops, bytes_ = kernel_work(dom[0])
    dur_s = dom[1][1] / dom[1][0] / 1e3
    tf, gbs = flops / dur_s / 1e12, bytes_ / dur_s / 1e9
    if tf / pk["bf16_tflops_sustained"] >= gbs / pk["hbm_gbs"]:
        roof = {"bound": "tensor", "achieved": tf, "peak": pk["bf16_tflops_sustained"], "unit": "TFLOP/s", "frac": tf / pk["bf16_tflops_sustained"]}
    else:
        roof = {"bound": "hbm", "achieved": gbs, "peak": pk["hbm_gbs"], "unit": "GB/s", "frac": gbs / pk["hbm_gbs"]}
    roof.update({"kernel": dom[0], "share_of_step": dom[1][1] / tot_prof, "avg_launch_ms": dur_s * 1e3,
                 "algorithmic_bytes": bytes_, "algorithmic_flops": flops,
                 "peak_source": pk["source"] + ", sustained bf16 figure (kernel timed inside a long step)"})
    ffwd = flop_fwd_per_impression(model_name, F)
    step_tf = value / world * 3 * ffwd / 1e12
    comp_bytes = bytes_per_impression(model_name)
    step_gbs = value / world * comp_bytes / 1e9
    breakdown = {k: round(v[1] / args.steps, 4) for k, v in sorted(prof.items(), key=lambda kv: -kv[1][1])}
    n_tok_bytes = sum(int(t.numel()) * 8 for d in (host_batches[0][1] + host_batches[0][2]) for t in d.values())
    out = {
        "metric": "impressions/sec (fwd+bwd)", "value": value, "unit": "impressions/s", "n_gpus": world, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": ms_total / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "bf16", "data": "synthetic",
        "config": {"workload": workload, "global_batch": B * world, "parallelism": f"dp{world}",
                   "l2": "3 rotating batches; per-step intermediates (> 1 GB) exceed the 50 MB L2", "dropout": 0.2,
                   "operand_refresh": "every step (bf16 table / weight shadows rebuilt as after an optimizer update)" if not args.no_operand_refresh else "off",
                   **({"precision": getattr(cfg, "precision", "fast")}
                      if model_name == "NRMS" else {})},
        "e2e": {"value": e2e, "unit": "impressions/s", "ms_per_step": ms_e2e / args.steps,
                "h2d_bytes_per_step": n_tok_bytes, "d2h_bytes_per_step": 4,
                "path": "model(candidate_news, clicked_news) with CPU slot lists (the call of the reference's train.py:202), loss.item() every step"},
        "gpu_launches": launches,
        "clocks": clk.summary(),
        "roofline": roof,
        "roofline_step": {"bound": "tensor", "achieved": step_tf, "peak": pk["bf16_tflops_sustained"], "unit": "TFLOP/s",
                          "frac": step_tf / pk["bf16_tflops_sustained"],
                          "hbm_compulsory": {"bytes_per_step": comp_bytes * B, "achieved_gbs": step_gbs, "frac": step_gbs / pk["hbm_gbs"]},
                          "note": "whole step per GPU: algorithmic 3 x %.1f MFLOP and %.2f MB compulsory HBM bytes per impression (SURVEY 8d) / step time"
                                  % (ffwd / 1e6, comp_bytes / 1e6)},
        "kernel_ms_per_step": breakdown,
    }
    if ms_pref is not None:
        out["e2e_prefetch"] = {"value": imp / (ms_pref / 1e3), "unit": "impressions/s", "ms_per_step": ms_pref / args.steps,
                               "path": "NRMS.prefetch stages the next batch on a copy stream (not a reference API)"}
    if world == 1 and not args.no_cpu_baseline:
        val, ms, cores, kind = run_reference(model_name, ref_batch, 2, 1, F)
        out["cpu_baseline"] = {"value": val, "unit": "impressions/s", "cores": cores, "kind": "port",
                               "sample": f"2 steps of {ref_batch} impressions after 1 warm-up (same shapes, same batch); {kind}; {ms:.0f} ms/step"}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    try:
        main()
    except BaseException:  # noqa: BLE001  (a failure must never look like an empty result)
        import traceback
        traceback.print_exc()
        sys.stderr.flush()
        raise
