"""Data parallel on real GPUs (NCCL): the gradient all-reduce that overlaps the backward must give exactly what two
independent single-GPU backward passes give when averaged.

The overlapped path is easy to get wrong silently: the backward records a CUDA event behind the embedding-gradient scatter
GEMM, `FlatGradients.all_reduce_mean` sends that slice from a side stream as soon as the event fires -- while the
weight-gradient GEMMs still run on 100 of the 132 SMs -- and reduces the rest afterwards (src/newsrec_b200/ddp.py,
csrc/abi.cu nr_mhsa_encoder_bwd).  An all-reduce that started before the scatter had finished, or a weight-gradient GEMM
that raced with it, would corrupt gradients without any error.  Needs two GPUs (skipped otherwise)."""
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _worker(rank, world, port, out_dir):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    for p in (os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle"), os.path.join(ROOT, "news-recommendation_b200", "src")):
        sys.path.insert(0, p)
    import gpu_checks as G
    import newsrec_oracle as O
    from newsrec_b200 import ddp
    torch.cuda.set_device(rank)
    G.DEV = torch.device("cuda", rank)
    r, w, _ = ddp.init_from_env("nccl")
    B, Cn, H, T, V = 16, 5, 50, 20, 3000
    model, _ = G.nrms_model_and_params(V, seed=3, fused="accurate")
    ref, _ = G.nrms_model_and_params(V, seed=3, fused="accurate")   # same weights, plain autograd gradients, no communication
    model.eval()  # no dropout: the two ranks differ only in their batches
    ref.eval()
    flat = ddp.FlatGradients(model.parameters(), w)
    name_of = {id(prm): k for k, prm in model.named_parameters()}
    ref_params = dict(ref.named_parameters())
    pad4 = lambda n: (n + 3) // 4 * 4
    label = torch.zeros(B, dtype=torch.long, device=G.DEV)
    results = []
    for step in range(3):  # several steps: the event / side stream are reused
        cand_t, clicked_t, _ = O.synth_batch(B, Cn, H, T, V, 100 * step + r)
        ref.zero_grad(set_to_none=True)
        torch.nn.functional.cross_entropy(ref(G.slots(cand_t), G.slots(clicked_t)), label).backward()
        local = torch.zeros_like(flat.flat)  # this rank's own gradient in the flat buffer's layout
        off = 0
        for prm in flat.params:
            n = prm.numel()
            local[off:off + n] = ref_params[name_of[id(prm)]].grad.reshape(-1)
            off += pad4(n)
        flat.zero()
        loss = torch.nn.functional.cross_entropy(model(G.slots(cand_t), G.slots(clicked_t)), label)
        loss.backward()
        flat.all_reduce_mean()  # no synchronisation in between: the slice all-reduce overlaps the weight-gradient GEMMs
        torch.cuda.synchronize()
        results.append((local.cpu(), flat.flat.clone().cpu()))
    torch.save(results, os.path.join(out_dir, f"rank{r}.pt"))
    torch.distributed.barrier()
    torch.distributed.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_overlapped_all_reduce_equals_the_mean_of_the_rank_gradients(tmp_path):
    import torch.multiprocessing as mp
    mp.spawn(_worker, args=(2, 29571, str(tmp_path)), nprocs=2, join=True)
    r0, r1 = torch.load(tmp_path / "rank0.pt"), torch.load(tmp_path / "rank1.pt")
    for step, ((l0, a0), (l1, a1)) in enumerate(zip(r0, r1)):
        assert torch.equal(a0, a1), f"step {step}: ranks disagree after the all-reduce"
        want = (l0.double() + l1.double()) / 2
        scale = float(want.abs().max())
        assert scale > 0
        err = float((a0.double() - want).abs().max()) / scale
        assert err < 2e-5, (step, err)  # fp32 atomics accumulate in a different order in the two replicas of a rank; nothing else differs
        assert float((l0 - l1).abs().max()) > 1e-3 * scale, "the two ranks must see different batches for the check to mean anything"
