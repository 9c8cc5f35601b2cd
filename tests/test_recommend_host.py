"""newsrec_b200.recommend without a GPU: the exclusion CSR, the line format and user order, the refusals raised before any
device work, and the CLI's argument parsing."""
import os

import numpy as np
import pytest

from newsrec_b200 import NewsrecError
from newsrec_b200 import recommend as R
from newsrec_b200.evaluate import distinct_histories, read_behaviors


def test_exclusion_csr_drops_padding_and_keeps_order():
    pad = 9
    hist = np.array([[pad, pad, 3, 4], [pad, pad, pad, pad], [1, 1, 2, 5], [pad, 0, pad, 8]])
    rows, offs = R.exclusion_csr(hist, pad)
    assert offs.tolist() == [0, 2, 2, 6, 8]
    assert rows.tolist() == [3, 4, 1, 1, 2, 5, 0, 8]           # the duplicate click is repeated, harmlessly
    assert rows.dtype == np.int64 and offs.dtype == np.int64
    rows, offs = R.exclusion_csr(np.zeros((0, 4), np.int64), pad)
    assert rows.size == 0 and offs.tolist() == [0]


def test_lines_and_user_order(tmp_path):
    import torch
    idx = torch.tensor([[2, 0, -1], [-1, -1, -1], [1, 2, 0]])
    text = R.format_lines(["U7", "U1", "U7"], idx.numpy(), ["N10", "N11", "N12"])
    assert text == b"U7\tN12,N10\nU1\t\nU7\tN11,N12,N10\n"
    d = str(tmp_path)
    with open(os.path.join(d, "behaviors.tsv"), "w") as f:
        f.write("1\tU2\tt\tN1 N2\tN3-1\n2\tU1\tt\t\tN3-0\n3\tU2\tt\tN1 N2\tN4-1\n4\tU3\tt\tN1 N2\tN4-1\n5\tU3\tt\tN5\tN4-1\n")
    users = distinct_histories(read_behaviors(d))["user"].tolist()
    assert users == ["U2", "U1", "U3"]                          # first appearance; the same history under U3 is U2's row


class _Cfg:
    num_clicked_news_a_user = 4


def _fake(name):
    return type(name, (), {"config": _Cfg})()


def test_refusals_come_before_the_device(tmp_path):
    d = str(tmp_path)
    for f in ("behaviors.tsv", "news_parsed.tsv"):
        open(os.path.join(d, f), "w").close()
    for k in (0, -3, 129, 2.5, True):
        with pytest.raises(NewsrecError, match="k="):
            R.check_request(_fake("NRMS"), d, k)
    for name, why in (("HiFiArk", "similarity attention"), ("DKN", "DNN click predictor")):
        with pytest.raises(NewsrecError, match=why):
            R.recommend(_fake(name), d, os.path.join(d, "out.tsv"), 10)
    for k in (1, 10, 128):
        R.check_request(_fake("NRMS"), d, k)
    os.remove(os.path.join(d, "behaviors.tsv"))
    with pytest.raises(FileNotFoundError, match="behaviors.tsv"):
        R.recommend(_fake("LSTUR"), d, os.path.join(d, "out.tsv"), 10)
    assert not os.path.exists(os.path.join(d, "out.tsv"))


def test_cli_arguments():
    a = R.parse_args(["--directory", "x", "--out", "y.tsv", "--k", "5", "--checkpoint", "c.pth", "--keep-clicked",
                      "--chunk-users", "3", "--set", "batch_size=2"])
    assert (a.directory, a.out, a.k, a.checkpoint, a.keep_clicked, a.chunk_users, a.set) == \
        ("x", "y.tsv", 5, "c.pth", True, 3, ["batch_size=2"])
    a = R.parse_args([])
    assert a.k == 10 and not a.keep_clicked and a.checkpoint is None and a.checkpoint_dir is None
    for bad in (["--k", "0"], ["--k", "129"], ["--chunk-users", "0"], ["--checkpoint", "a", "--checkpoint-dir", "b"]):
        with pytest.raises(SystemExit):
            R.parse_args(bad)
