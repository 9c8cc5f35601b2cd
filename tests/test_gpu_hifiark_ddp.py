"""Hi-Fi Ark under FlatGradients, the gradient storage `newsrec_b200.launch` trains with.  The archive kernels then add dW,
dW1, db1, dw2 and db2 straight into the parameters' `.grad` views (ops.grad_sink) and return None to autograd, a different
code path from the plain one; both must give the same gradients, and `abstract_CNN` (never read) must stay a zero view
that an Adam step leaves bit-identical.  Data parallel: the all-reduce of a Hi-Fi Ark step equals the mean of the ranks'
own gradients (NCCL on two GPUs, as tests/test_gpu_ddp.py does for NRMS; skipped with fewer)."""
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
V, B, C, H, T = 3000, 16, 5, 50, 20


def _model(dev):
    import config
    from model.HiFiArk import HiFiArk
    # dropout 0 in train mode: the regulariser runs, and two models see the same masks (none)
    cfg = type("Cfg", (config.HiFiArkConfig,), dict(num_words=V, num_clicked_news_a_user=H, dropout_probability=0.0))
    torch.manual_seed(3)
    return HiFiArk(cfg).to(dev).train()


def _step(model, seed, dev):
    import newsrec_oracle as O
    cand_t, clicked_t, _ = O.synth_batch(B, C, H, T, V, seed)
    slots = lambda t: [{"title": t[:, j].contiguous()} for j in range(t.shape[1])]
    logits, reg = model(slots(cand_t), slots(clicked_t))
    label = torch.zeros(B, dtype=torch.long, device=dev)
    (torch.nn.functional.cross_entropy(logits, label) + model.config.regularizer_loss_weight * reg).backward()


def test_flat_gradients_match_the_plain_path_and_leave_abstract_cnn_alone():
    from newsrec_b200 import ddp
    dev = torch.device("cuda", 0)
    plain, flat_model = _model(dev), _model(dev)
    flat_model.load_state_dict(plain.state_dict())
    flat = ddp.FlatGradients(flat_model.parameters(), 1)
    for step in range(2):  # the second step accumulates onto cleared views, as a training loop does
        plain.zero_grad(set_to_none=True)
        flat.zero()
        _step(plain, 10 + step, dev)
        _step(flat_model, 10 + step, dev)
        torch.cuda.synchronize()
        ref = dict(plain.named_parameters())
        for k, prm in flat_model.named_parameters():
            if k.startswith("news_encoder.abstract_CNN"):
                assert ref[k].grad is None and not prm.grad.any(), k
                continue
            want, got = ref[k].grad.double(), prm.grad.double()
            scale = float(want.abs().max())
            assert scale > 0, k
            # the archive and DNN gradients are summed in a fixed order (bit-identical); the news encoder's embedding scatter
            # accumulates with fp32 atomics, whose order differs between the two models
            assert float((got - want).abs().max()) <= 2e-5 * scale, (step, k)
    before = {k: v.detach().clone() for k, v in flat_model.news_encoder.abstract_CNN.named_parameters()}
    torch.optim.Adam(flat_model.parameters(), lr=1e-3).step()
    for k, v in flat_model.news_encoder.abstract_CNN.named_parameters():
        assert torch.equal(v.detach(), before[k]), k
    assert not torch.equal(flat_model.omap.W.detach(), plain.omap.W.detach())  # the step did move the parameters in use


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
    mp.spawn(_worker, args=(2, 29573, str(tmp_path)), nprocs=2, join=True)
    r0, r1 = torch.load(tmp_path / "rank0.pt"), torch.load(tmp_path / "rank1.pt")
    for step, ((l0, a0), (l1, a1)) in enumerate(zip(r0, r1)):
        assert torch.equal(a0, a1), f"step {step}: ranks disagree after the all-reduce"
        want = (l0.double() + l1.double()) / 2
        scale = float(want.abs().max())
        assert scale > 0
        err = float((a0.double() - want).abs().max()) / scale
        assert err < 2e-5, (step, err)  # the embedding scatter's fp32 atomics accumulate in a different order per replica
        assert float((l0 - l1).abs().max()) > 1e-3 * scale, "the two ranks must see different batches for the check to mean anything"
