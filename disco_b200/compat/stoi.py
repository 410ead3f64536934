"""Stands for pystoi.stoi (the ``stoi`` the reference imports at tango.py:23): stoi(x, y, fs_sig) with its NumPy-in /
float-out signature and its errors, computed by the float64 kernels of csrc/stoi.cu on the current CUDA device.  The
signals are rounded to float32 on the way in (the reference's signals are float32)."""
import numpy as np
import torch

from .. import stoi as _stoi


def stoi(x, y, fs_sig, extended=False):
    """pystoi.stoi.stoi: classic STOI of the 1-D clean x and degraded y at fs_sig Hz.  Raises Exception when the
    shapes differ and ValueError when fewer than 256 samples remain at 10 kHz, as pystoi does; extended=True (ESTOI)
    raises NotImplementedError."""
    x, y = np.asarray(x), np.asarray(y)
    if x.shape != y.shape:
        raise Exception("x and y should have the same length, found {} and {}".format(x.shape, y.shape))
    if extended:
        raise NotImplementedError("stoi: extended=True (ESTOI) is not implemented")
    if x.ndim != 1:
        raise ValueError("stoi: x and y must be 1-D, got shape {}".format(x.shape))
    dev = torch.device("cuda", torch.cuda.current_device())
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(dev)
    return float(_stoi.stoi(t(x), t(y), fs_sig).item())
