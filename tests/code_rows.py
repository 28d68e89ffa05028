"""Helpers for tests of the packed-code stores (SQ and MinMax), whose canonical rows end in dense N-bit codes."""
import numpy as np


def garbage_padding(rows, dim, nbits):
    """The rows with every bit past dim * nbits in the last code byte set."""
    tail = (dim * nbits) % 8
    out = rows.copy()
    if tail:
        out[:, -1] |= np.uint8((0xFF << tail) & 0xFF)
    return out
