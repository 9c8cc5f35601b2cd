"""Where do the gemm_nt CTAs spend their time?  One NRMS training step at the bench size with the per-role cycle counters
of nr_debug_set_gemm_timing switched on; prints, per GEMM launch, the share of the kernel each role (producer, each
consumer warpgroup's MMA turn wait, MMA loop and epilogue) took.

    python tools/gemm_timing.py [NRMS|NAML|LSTUR|TANR] [batch]
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "news-recommendation_b200", "src"))

import torch  # noqa: E402

import importlib  # noqa: E402

import bench  # noqa: E402
import config as cfgmod  # noqa: E402
import newsrec_b200  # noqa: E402

args = [a for a in sys.argv[1:]]
name = args[0] if args and not args[0].isdigit() else "NRMS"
B = int(args[-1]) if args and args[-1].isdigit() else 512
dev = torch.device("cuda", 0)
lib = newsrec_b200.load_library()
Model = getattr(importlib.import_module("model." + name), name)
over = {"long_short_term_method": "ini"} if name == "LSTUR" else {}
model = Model(type("Cfg", (getattr(cfgmod, name + "Config"),), over)).to(dev)
model.train()
extra, cand, clicked = bench.synth_slots(name, B, 7, device=dev)
label = torch.zeros(B, dtype=torch.long, device=dev)


def step():
    model.zero_grad(set_to_none=True)
    out = model(extra[0], extra[1].clone(), cand, clicked) if name == "LSTUR" else model(cand, clicked)
    loss = torch.nn.functional.cross_entropy(out[0], label) + 0.1 * out[1] if isinstance(out, tuple) else torch.nn.functional.cross_entropy(out, label)
    loss.backward()
    torch.cuda.synchronize()


for _ in range(2):
    step()
SLOTS = 32
buf = torch.zeros(SLOTS, 148, 16, dtype=torch.int64, device=dev)
lib.nr_debug_set_gemm_timing(buf.data_ptr(), SLOTS)
step()
lib.nr_debug_set_gemm_timing(None, 0)
t = buf.cpu().double()
# per CTA (gemm_nt_kernel): [0] producer waits for a free stage, [1] weight slice, [5] kernel; consumer warpgroup w at
# [8 + 4w]: +0 waits for its MMA turn, +1 MMA loops (waits for A data included), +2 epilogue, +3 tiles.  With the epilogue
# overlapped, mma0 + mma1 approaches 100% of the kernel while each warpgroup's epilogue share stays large.
for s in range(SLOTS):
    used = t[s, :, 5] > 0
    if used.sum() == 0:
        continue
    m = t[s][used].mean(0)
    k = m[5].item()
    pct = lambda i: 100 * m[i].item() / k
    wgs = "  ".join(f"wg{w}: turn={pct(8 + 4 * w):5.1f}% mma={pct(9 + 4 * w):5.1f}% epi={pct(10 + 4 * w):5.1f}% "
                    f"tiles={m[11 + 4 * w].item():6.1f} epi/tile={m[10 + 4 * w].item() / max(m[11 + 4 * w].item(), 1):6.0f} cyc"
                    for w in range(2))
    print(f"slot {s:2d} ctas={int(used.sum())} kernel={k / 1e3:8.1f} kcyc prod:empty={pct(0):5.1f}%  {wgs}", flush=True)
    # per weight slice: the CTAs of one slice share its column range, so an epilogue that costs more on some columns (the
    # low plane of the accurate V section) shows up as a slice whose CTAs run longer
    slices = t[s, :, 1][used]
    if int(slices.max()) == 0:
        continue
    for sl in range(int(slices.max()) + 1):
        c = t[s][used][slices == sl]
        tiles = c[:, 11] + c[:, 15]
        print(f"         slice {sl}: ctas={c.shape[0]:3d} kernel={c[:, 5].mean().item() / 1e3:8.1f} kcyc "
              f"(max {c[:, 5].max().item() / 1e3:8.1f})  mma/tile={(c[:, 9] + c[:, 13]).sum().item() / max(tiles.sum().item(), 1):6.0f} cyc "
              f"epi/tile={(c[:, 10] + c[:, 14]).sum().item() / max(tiles.sum().item(), 1):6.0f} cyc", flush=True)
