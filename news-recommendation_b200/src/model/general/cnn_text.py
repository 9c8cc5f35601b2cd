"""Shared host-side pieces of the CNN text encoders (NAML / LSTUR / TANR / Hi-Fi Ark)."""
import torch
import torch.nn as nn

from newsrec_b200 import NewsrecError, require_cuda
from newsrec_b200.guard import BadIdFlag  # noqa: F401  (re-exported: the CNN model packages import it from here)
from newsrec_b200.ops import OperandCache
from newsrec_b200.ops_cnn import CnnPoolEncoderFn

CNN_WINDOWS = (1, 2, 3, 4)  # the conv windows the encoder kernels run (include/newsrec_b200.h)


def make_title_cnn(num_filters, window_size, word_embedding_dim):
    """Parameter container with the reference's shapes: weight (F, 1, window, d), bias (F).  A window the kernels do not run
    is refused here, when the model is built, rather than at the first batch."""
    if window_size not in CNN_WINDOWS:
        raise NewsrecError(f"window_size={window_size!r}: the CNN text encoders run windows 1 to 4 (include/newsrec_b200.h)")
    return nn.Conv2d(1, num_filters, (window_size, word_embedding_dim), padding=(int((window_size - 1) / 2), 0))


def cnn_text_encode(ids, word_embedding, cnn, attention, p_drop, cache: OperandCache, prefix, flag: BadIdFlag, accurate=False):
    """ids (n, T) int64 on the device -> (n, F) through the fused gather/conv/ReLU/pool kernel sequence."""
    dev = require_cuda()
    return CnnPoolEncoderFn.apply(ids, word_embedding.weight, cnn.weight, cnn.bias, attention.linear.weight,
                                  attention.linear.bias, attention.attention_query_vector, p_drop, cache, prefix,
                                  flag.get(dev), bool(accurate))
