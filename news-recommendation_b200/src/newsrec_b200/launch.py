"""Data-parallel launcher around the reference's UNMODIFIED `src/train.py` (SURVEY.md section 8f, row N1).

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 \\
        -m newsrec_b200.launch --reference-src /path/to/news-recommendation/src

Run from the directory that holds `./data` exactly as the reference expects (`train.py` uses cwd-relative paths).  Every
rank imports the reference trainer with the drop-in `model.*` / `config` packages shadowing the reference's, and calls
`train.train()`.  The reference loop (train.py:67-279) is single-process; what this module changes around it, without
editing it:

* one GPU per process: `CUDA_VISIBLE_DEVICES` is narrowed to LOCAL_RANK before CUDA initialises, so the reference's
  `cuda:0` (train.py:24) is this rank's GPU;
* `DataLoader(..., shuffle=True)` (train.py:119, :173) becomes a `DistributedSampler` over the same dataset (disjoint
  shards, a new permutation every time the reference re-creates the loader);
* `torch.optim.Adam` (train.py:127) becomes `AllReduceAdam`: gradients live in one flat fp32 buffer
  (`ddp.FlatGradients`: the kernels accumulate into it in place), `zero_grad()` clears that buffer, `step()` first
  all-reduces it (ONE NCCL collective, mean over ranks) -- every rank then applies the identical update;
* rank 0 alone writes TensorBoard events and checkpoints and runs `evaluate()` (train.py:248); its metrics are broadcast
  so that early stopping takes the same decision everywhere; `--device-evaluate` swaps the reference's evaluator for
  `newsrec_b200.evaluate.evaluate` (same signature; scoring and metrics on the device);
* `--device-feed` replaces the trainer's `BaseDataset` with `newsrec_b200.feed.DeviceFeed` (tables parsed once and held on
  the device, one gather launch per batch; SURVEY.md row N3); the DataLoader factory returns the feed's loader for it,
  over the same sharding, seed and epoch counter; `--resample-negatives` makes it a feed over the raw behaviors.tsv
  whose negatives are redrawn on the device every epoch from `--seed` and that epoch counter (the same on every rank);
* compatibility shims the survey found necessary for the reference on current NumPy / pandas / torch.
"""
from __future__ import annotations

import argparse
import functools
import os
import sys


def _env_int(name, default):
    return int(os.environ.get(name, default))


class _NullWriter:
    """SummaryWriter stand-in for ranks != 0."""

    def __init__(self, *a, **k):
        pass

    def __getattr__(self, name):
        return lambda *a, **k: None


def make_sharded_dataloader(base_loader_cls, rank, world, seed=0):
    """DataLoader factory with the reference's call signature; `shuffle=True` turns into a DistributedSampler."""
    import torch
    from torch.utils.data.distributed import DistributedSampler

    state = {"epoch": 0}

    def factory(dataset, *args, **kwargs):
        if world > 1 and kwargs.get("sampler") is None and kwargs.get("batch_sampler") is None:
            shuffle = bool(kwargs.pop("shuffle", False))
            sampler = DistributedSampler(dataset, num_replicas=world, rank=rank, shuffle=shuffle, seed=seed,
                                         drop_last=bool(kwargs.get("drop_last", False)))
            sampler.set_epoch(state["epoch"])  # the reference builds a fresh loader each time the data is exhausted
            state["epoch"] += 1
            kwargs["sampler"] = sampler
        if not torch.cuda.is_available():
            kwargs.pop("pin_memory", None)
        return base_loader_cls(dataset, *args, **kwargs)

    return factory


def make_feed_dataloader(base_factory, rank, world, seed=0):
    """DataLoader factory that hands a DeviceFeed its own loader (rows sharded by a DistributedSampler with `seed`, a new
    epoch each time the trainer re-creates the loader) and every other dataset to `base_factory`."""
    from newsrec_b200.feed import DeviceFeed

    state = {"epoch": 0}

    def factory(dataset, *args, **kwargs):
        if not isinstance(dataset, DeviceFeed):
            return base_factory(dataset, *args, **kwargs)
        loader = dataset.loader(kwargs.get("batch_size", args[0] if args else 1), shuffle=kwargs.get("shuffle", False),
                                drop_last=kwargs.get("drop_last", False), rank=rank, world=world, seed=seed, epoch=state["epoch"])
        state["epoch"] += 1
        return loader

    return factory


def make_all_reduce_adam(base_adam_cls, world):
    """Adam whose gradients live in ddp.FlatGradients and are all-reduced (mean) right before every step."""
    from newsrec_b200 import ddp

    class AllReduceAdam(base_adam_cls):
        def __init__(self, params, *args, **kwargs):
            params = list(params)
            flat_params = []
            for p in params:  # plain parameter list or param groups
                flat_params.extend(p["params"] if isinstance(p, dict) else [p])
            self._flat = ddp.FlatGradients(flat_params, world)
            super().__init__(params, *args, **kwargs)

        def zero_grad(self, set_to_none=True):  # keep the views: the kernels accumulate into them in place
            self._flat.zero()

        def step(self, closure=None):
            self._flat.all_reduce_mean()
            return super().step(closure)

    return AllReduceAdam


def make_rank0_evaluate(evaluate_fn, rank, world):
    """evaluate() runs on rank 0 only; the metrics are broadcast so that every rank sees the same early-stop signal."""
    import torch.distributed as dist

    def wrapped(*args, **kwargs):
        box = [evaluate_fn(*args, **kwargs) if rank == 0 else None]
        if world > 1:
            dist.broadcast_object_list(box, src=0)
        return box[0]

    return wrapped


def apply_compat_shims():
    """Environment-version shims for the reference's drivers (SURVEY.md 8c): NumPy 2 removed np.Inf (train.py:31),
    pandas 3 infers str columns (evaluate.py:99), torch >= 2.6 defaults torch.load to weights_only=True while the
    reference checkpoints hold a numpy scalar (train.py:147, :275)."""
    import numpy as np
    if not hasattr(np, "Inf"):
        np.Inf = np.inf
    try:
        import pandas as pd
        pd.options.future.infer_string = False
    except Exception:  # pandas absent or option renamed: the trainer itself does not need it
        pass
    import torch
    if not getattr(torch.load, "_newsrec_patched", False):
        _load = torch.load

        def load(*a, **k):
            k.setdefault("weights_only", False)
            return _load(*a, **k)

        load._newsrec_patched = True
        torch.load = load


def patch_trainer(train_module, rank, world, seed=0, device_evaluate=False, device_feed=False, resample_negatives=False):
    """Install the data-parallel pieces into an imported (reference) `train` module's namespace.  device_evaluate: the
    trainer's `evaluate` becomes newsrec_b200.evaluate.evaluate (its docstring lists where its metrics can differ from a
    given reference environment: ties across labels, one-class impressions).  device_feed: the trainer's `BaseDataset`
    becomes newsrec_b200.feed.DeviceFeed and its DataLoader returns the feed's loader for it.  resample_negatives (with
    device_feed): that feed reads data/train/behaviors.tsv and redraws its negatives per (seed, epoch)."""
    import torch
    train_module.DataLoader = make_sharded_dataloader(train_module.DataLoader, rank, world, seed)
    if device_feed:
        from newsrec_b200.feed import DeviceFeed
        train_module.BaseDataset = functools.partial(DeviceFeed, resample_negatives=True, seed=seed) if resample_negatives else DeviceFeed
        train_module.DataLoader = make_feed_dataloader(train_module.DataLoader, rank, world, seed)
    if world > 1 or os.environ.get("NEWSREC_FLAT_GRADS", "1") == "1":
        # the trainer reaches Adam through the global `torch.optim` module (train.py:127)
        torch.optim.Adam = make_all_reduce_adam(torch.optim.Adam, world)
    if device_evaluate:
        from newsrec_b200.evaluate import evaluate as device_evaluate_fn
        train_module.evaluate = make_rank0_evaluate(device_evaluate_fn, rank, world)
    elif hasattr(train_module, "evaluate"):
        train_module.evaluate = make_rank0_evaluate(train_module.evaluate, rank, world)
    if rank != 0:
        if hasattr(train_module, "SummaryWriter"):
            train_module.SummaryWriter = _NullWriter
        _save = torch.save
        torch.save = lambda *a, **k: None  # checkpoints are rank 0's job
        torch.save._newsrec_original = _save


def set_knobs(items):
    """Apply KNOB=VALUE strings to the selected <MODEL_NAME>Config (VALUE read as a Python literal, else kept as the
    string); returns the config class."""
    import ast
    import importlib
    cfgmod = importlib.import_module("config")
    cfg = getattr(cfgmod, f"{cfgmod.model_name}Config")
    for item in items:
        key, _, val = item.partition("=")
        try:
            val = ast.literal_eval(val)
        except (ValueError, SyntaxError):
            pass  # keep the string
        setattr(cfg, key, val)
    return cfg


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reference-src", required=True, help="the reference repository's src/ directory (train.py, dataset.py, evaluate.py)")
    ap.add_argument("--no-dropin", action="store_true", help="keep the reference's own model/config packages (CPU smoke runs)")
    ap.add_argument("--backend", default=None, help="torch.distributed backend (default: nccl with CUDA, else gloo)")
    ap.add_argument("--seed", type=int, default=0, help="seed of the sharded sampler's permutations")
    ap.add_argument("--device-evaluate", action="store_true",
                    help="validate with newsrec_b200.evaluate.evaluate (all impressions scored and their AUC / MRR / nDCG computed "
                         "on the device) instead of the reference's evaluate.py")
    ap.add_argument("--device-feed", action="store_true",
                    help="train from newsrec_b200.feed.DeviceFeed: news and behaviour tables parsed once and kept on the device, "
                         "every batch gathered there by one kernel launch instead of the reference's BaseDataset / DataLoader")
    ap.add_argument("--resample-negatives", action="store_true",
                    help="with --device-feed: train on MIND's raw behaviors.tsv and redraw each impression's negatives on the device "
                         "every epoch (seeded by --seed) instead of the fixed draw in behaviors_parsed.tsv")
    ap.add_argument("--set", action="append", default=[], metavar="KNOB=VALUE",
                    help="override a knob of the selected <MODEL_NAME>Config before the trainer is imported (repeatable), "
                         "e.g. --set batch_size=512 --set num_workers=8")
    args = ap.parse_args(argv)
    if args.resample_negatives and not args.device_feed:
        ap.error("--resample-negatives needs --device-feed")

    rank, world, local = _env_int("RANK", 0), _env_int("WORLD_SIZE", 1), _env_int("LOCAL_RANK", 0)
    # the ranks share one stdout pipe: with block buffering a flush can end mid-line and another rank's output then lands
    # inside that line (train.py's loss lines run together); line buffering makes every line one write, which a pipe keeps whole
    if world > 1 and hasattr(sys.stdout, "reconfigure"):
        sys.stdout.reconfigure(line_buffering=True)
    if "CUDA_VISIBLE_DEVICES" not in os.environ or os.environ.get("NEWSREC_PIN_GPU", "1") == "1":
        vis = os.environ.get("CUDA_VISIBLE_DEVICES")
        if vis is None:
            os.environ["CUDA_VISIBLE_DEVICES"] = str(local)
        else:
            ids = [v for v in vis.split(",") if v != ""]
            if len(ids) > 1 and local < len(ids):
                os.environ["CUDA_VISIBLE_DEVICES"] = ids[local]
    if rank != 0:
        os.environ.setdefault("TQDM_DISABLE", "1")

    here = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))  # .../news-recommendation_b200/src
    from newsrec_b200 import ddp  # noqa: F401  (resolved now: --no-dropin takes the package's directory off the path below)
    sys.path.insert(0, os.path.abspath(args.reference_src))
    if not args.no_dropin:
        sys.path.insert(0, here)  # model.*, config shadow the reference's
    else:
        # the reference's `model` is a namespace package (no __init__.py): a regular package of the same name anywhere
        # on the path would win over it, so the drop-in's directory must not be on the path at all
        sys.path[:] = [q for q in sys.path if os.path.abspath(q or os.getcwd()) != here]
    apply_compat_shims()

    import torch
    import torch.distributed as dist
    if world > 1 and not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29511")
        backend = args.backend or ("nccl" if torch.cuda.is_available() else "gloo")
        # rank 0 alone runs the reference's evaluate() (a Python loop over up to 200k impressions) while the other ranks
        # already wait in the next collective: the default 10-minute NCCL watchdog would abort the job
        import datetime
        dist.init_process_group(backend=backend, rank=rank, world_size=world, timeout=datetime.timedelta(hours=6))

    import importlib
    if args.set:
        set_knobs(args.set)
    train = importlib.import_module("train")
    feed = {"device_feed": True} if args.device_feed else {}  # without the flag: the call (and the patch) of before
    if args.resample_negatives:
        feed["resample_negatives"] = True
    patch_trainer(train, rank, world, args.seed, device_evaluate=args.device_evaluate, **feed)
    try:
        train.train()
    finally:
        if world > 1 and dist.is_initialized():
            dist.barrier()
            dist.destroy_process_group()


if __name__ == "__main__":
    main()
