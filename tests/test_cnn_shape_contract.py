"""nr_cnn_encoder_fwd / _bwd reject the shapes their kernels do not cover with -1 before any launch (include/newsrec_b200.h):
segments longer than one 64-row pooling tile and filter counts that are not a multiple of 4.  The check runs before any
pointer or device is touched, so it runs without a GPU."""
import ctypes

import pytest


def _lib():
    import newsrec_b200
    import os
    if not os.path.exists(newsrec_b200.LIB_PATH):
        pytest.skip("library not built (python __graft_entry__.py build)")
    return newsrec_b200.load_library()


def _ru8(x):
    return (x + 7) // 8 * 8


def _call(which, T, F, d=300, q=200):
    import newsrec_b200 as nb
    lib = _lib()
    a = nb.CnnEncoderFwdArgs() if which == "fwd" else nb.CnnEncoderBwdArgs()
    a.n_seq, a.T, a.d, a.F, a.q, a.ldx, a.ldf = 8, T, d, F, q, _ru8(d + 1), _ru8(F + 1)
    if which == "bwd":
        a.ldq = (q + 15) // 16 * 16
    n0 = lib.nr_launch_count()
    fn = lib.nr_cnn_encoder_fwd if which == "fwd" else lib.nr_cnn_encoder_bwd
    rc = fn(ctypes.byref(a), None)
    return rc, lib.nr_last_error().decode(), lib.nr_launch_count() - n0


@pytest.mark.parametrize("which", ["fwd", "bwd"])
@pytest.mark.parametrize("T", [65, 126])
def test_segments_longer_than_a_pooling_tile_are_rejected_before_launch(which, T):
    rc, msg, launched = _call(which, T, 400)
    assert rc == -1 and f"T={T}" in msg and launched == 0, (rc, msg, launched)


@pytest.mark.parametrize("which", ["fwd", "bwd"])
def test_filter_count_not_a_multiple_of_4_is_rejected_before_launch(which):
    rc, msg, launched = _call(which, 20, 250)
    assert rc == -1 and "F=250" in msg and launched == 0, (rc, msg, launched)


@pytest.mark.parametrize("which", ["fwd", "bwd"])
def test_longest_segment_passes_the_shape_check(which):
    """T = 64 is accepted: with null operands the call fails on the pointers instead, still before any launch."""
    rc, msg, launched = _call(which, 64, 400)
    assert rc == -1 and "null operand" in msg and launched == 0, (rc, msg, launched)
