"""DKN under FlatGradients, the gradient storage `newsrec_b200.launch` trains with: every parameter's `.grad` is a view into one
flat buffer that autograd accumulates into, a different code path from the plain one; both must give the same gradients over
two steps, at the default windows and at a repeated window, where one conv parameter receives two gradient contributions in
one backward.  The gradients of the candidate half of attention.dnn.0.weight and of both attention biases are exact zeros
(the softmax over the history cancels them) in the flat views too.  Data parallel: the all-reduce of a DKN step equals the
mean of the ranks' own gradients (NCCL on two GPUs, as tests/test_gpu_hifiark_ddp.py does; skipped with fewer)."""
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
V, VE, B, C, H, T = 3000, 400, 16, 5, 50, 20
DEAD = ("attention.dnn.0.bias", "attention.dnn.1.bias")


def _model(dev, windows=(2, 3, 4)):
    import config
    from model.DKN import DKN
    cfg = type("Cfg", (config.DKNConfig,), dict(num_words=V, num_entities=VE, num_clicked_news_a_user=H, window_sizes=list(windows)))
    torch.manual_seed(3)
    return DKN(cfg).to(dev).train()  # DKN has no dropout


def _step(model, seed, dev):
    import dkn_oracle as DO
    import newsrec_oracle as O
    cand_t, clicked_t, _ = O.synth_batch(B, C, H, T, V, seed)
    cand_e, clicked_e = DO.synth_entities(cand_t, VE, seed + 50), DO.synth_entities(clicked_t, VE, seed + 60)
    slots = lambda t, e: [{"title": t[:, j].contiguous(), "title_entities": e[:, j].contiguous()} for j in range(t.shape[1])]
    logits = model(slots(cand_t, cand_e), slots(clicked_t, clicked_e))
    torch.nn.functional.cross_entropy(logits, torch.zeros(B, dtype=torch.long, device=dev)).backward()


@pytest.mark.parametrize("windows", [(2, 3, 4), (3, 3)], ids=["w234", "w33"])
def test_flat_gradients_match_the_plain_path(windows):
    from newsrec_b200 import ddp
    dev = torch.device("cuda", 0)
    plain, flat_model = _model(dev, windows), _model(dev, windows)
    flat_model.load_state_dict(plain.state_dict())
    flat = ddp.FlatGradients(flat_model.parameters(), 1)
    Fp = 50 * len(windows)
    for step in range(2):  # the second step accumulates onto cleared views, as a training loop does
        plain.zero_grad(set_to_none=True)
        flat.zero()
        _step(plain, 10 + step, dev)
        _step(flat_model, 10 + step, dev)
        torch.cuda.synchronize()
        ref = dict(plain.named_parameters())
        for k, prm in flat_model.named_parameters():
            want, got = ref[k].grad.double(), prm.grad.double()
            if k in DEAD:
                assert not got.any() and not want.any(), (step, k)
                continue
            if k == "attention.dnn.0.weight":
                assert not got[:, :Fp].any() and not want[:, :Fp].any(), step
            scale = float(want.abs().max())
            assert scale > 0, k
            # the user kernels and the scorer sum in a fixed order; the encoder's embedding scatters accumulate with fp32
            # atomics, whose order differs between the two models
            assert float((got - want).abs().max()) <= 2e-5 * scale, (step, k)
            assert prm.grad.data_ptr() >= flat.flat.data_ptr() and \
                prm.grad.data_ptr() < flat.flat.data_ptr() + 4 * flat.flat.numel(), k  # still the flat view


def _worker(rank, world, port, out_dir):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    for p in (os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle"), os.path.join(ROOT, "news-recommendation_b200", "src")):
        sys.path.insert(0, p)
    from newsrec_b200 import ddp
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    r, w, _ = ddp.init_from_env("nccl")
    model, ref = _model(dev), _model(dev)  # same weights; ref: plain autograd gradients, no communication
    ref.load_state_dict(model.state_dict())
    flat = ddp.FlatGradients(model.parameters(), w)
    name_of = {id(prm): k for k, prm in model.named_parameters()}
    ref_params = dict(ref.named_parameters())
    pad4 = lambda n: (n + 3) // 4 * 4
    results = []
    for step in range(3):
        ref.zero_grad(set_to_none=True)
        _step(ref, 100 * step + r, dev)
        local = torch.zeros_like(flat.flat)
        off = 0
        for prm in flat.params:
            n = prm.numel()
            g = ref_params[name_of[id(prm)]].grad
            if g is not None:
                local[off:off + n] = g.reshape(-1)
            off += pad4(n)
        flat.zero()
        _step(model, 100 * step + r, dev)
        flat.all_reduce_mean()
        torch.cuda.synchronize()
        results.append((local.cpu(), flat.flat.clone().cpu()))
    torch.save(results, os.path.join(out_dir, f"rank{r}.pt"))
    torch.distributed.barrier()
    torch.distributed.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_all_reduce_equals_the_mean_of_the_rank_gradients(tmp_path):
    import torch.multiprocessing as mp
    mp.spawn(_worker, args=(2, 29581, str(tmp_path)), nprocs=2, join=True)
    r0, r1 = torch.load(tmp_path / "rank0.pt"), torch.load(tmp_path / "rank1.pt")
    for step, ((l0, a0), (l1, a1)) in enumerate(zip(r0, r1)):
        assert torch.equal(a0, a1), f"step {step}: ranks disagree after the all-reduce"
        want = (l0.double() + l1.double()) / 2
        scale = float(want.abs().max())
        assert scale > 0
        err = float((a0.double() - want).abs().max()) / scale
        assert err < 2e-5, (step, err)  # the embedding scatters' fp32 atomics accumulate in a different order per replica
        assert float((l0 - l1).abs().max()) > 1e-3 * scale, "the two ranks must see different batches for the check to mean anything"
