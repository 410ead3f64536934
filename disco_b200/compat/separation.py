"""Stands for mir_eval.separation (the ``bss`` the reference imports at tango.py:22): bss_eval_sources with its
NumPy-in / NumPy-out signature and its input validation, computed by the float64 kernels of csrc/bss.cu on the
current CUDA device.  The signals are rounded to float32 on the way in (the reference's signals are float32)."""
import numpy as np
import torch

from .. import bss_eval as _bss

MAX_SOURCES = 100   # mir_eval's limit; the kernels take up to 4 (more raise NotImplementedError)


def _any_source_silent(sources):
    return np.any(np.all(np.sum(sources, axis=tuple(range(2, sources.ndim))) == 0, axis=1))


def validate(reference_sources, estimated_sources):
    """mir_eval.separation.validate: ValueError for mismatched shapes, more than 3 dimensions, all-zero sources or
    more than MAX_SOURCES sources; an empty input only warns."""
    import warnings
    if reference_sources.shape != estimated_sources.shape:
        raise ValueError("The shape of estimated sources and the true sources should match.  reference_sources.shape "
                         "= {}, estimated_sources.shape = {}".format(reference_sources.shape, estimated_sources.shape))
    if reference_sources.ndim > 3 or estimated_sources.ndim > 3:
        raise ValueError("The number of dimensions is too high (must be less than 3). reference_sources.ndim = {}, "
                         "estimated_sources.ndim = {}".format(reference_sources.ndim, estimated_sources.ndim))
    if reference_sources.size == 0:
        warnings.warn("reference_sources is empty, should be of size (nsrc, nsample).  sdr, sir, sar, and perm will "
                      "all be empty np.ndarrays")
    elif _any_source_silent(reference_sources):
        raise ValueError("All the reference sources should be non-silent (not all-zeros), but at least one of the "
                         "reference sources is all 0s, which introduces ambiguity to the evaluation. (Otherwise we can "
                         "add infinitesimal noise?)")
    if estimated_sources.size == 0:
        warnings.warn("estimated_sources is empty, should be of size (nsrc, nsample).  sdr, sir, sar, and perm will "
                      "all be empty np.ndarrays")
    elif _any_source_silent(estimated_sources):
        raise ValueError("All the estimated sources should be non-silent (not all-zeros), but at least one of the "
                         "estimated sources is all 0s. Since we require each reference source to be non-silent, having "
                         "a silent estimated source will result in an underdetermined system.")
    if estimated_sources.shape[0] > MAX_SOURCES or reference_sources.shape[0] > MAX_SOURCES:
        raise ValueError("The supplied matrices should be of shape (nsrc, nsampl) but reference_sources.shape[0] = {} "
                         "and estimated_sources.shape[0] = {} which is greater than mir_eval.separation.MAX_SOURCES = "
                         "{}.  To override this check, set mir_eval.separation.MAX_SOURCES to a larger value.".format(
                             reference_sources.shape[0], estimated_sources.shape[0], MAX_SOURCES))


def bss_eval_sources(reference_sources, estimated_sources, compute_permutation=True):
    """mir_eval.separation.bss_eval_sources: (nsrc, nsampl) arrays (1-D = one source) -> sdr, sir, sar (float64) and
    perm (int64), each of length nsrc."""
    reference_sources = np.asarray(reference_sources)
    estimated_sources = np.asarray(estimated_sources)
    if estimated_sources.ndim == 1:
        estimated_sources = estimated_sources[np.newaxis, :]
    if reference_sources.ndim == 1:
        reference_sources = reference_sources[np.newaxis, :]
    validate(reference_sources, estimated_sources)
    if reference_sources.size == 0 or estimated_sources.size == 0:
        return np.array([]), np.array([]), np.array([]), np.array([])
    if reference_sources.ndim != 2:
        raise NotImplementedError("bss_eval_sources: multichannel (3-D) sources are not supported")
    dev = torch.device("cuda", torch.cuda.current_device())
    refs = torch.from_numpy(np.ascontiguousarray(reference_sources, dtype=np.float32)).to(dev)
    ests = torch.from_numpy(np.ascontiguousarray(estimated_sources, dtype=np.float32)).to(dev)
    out = _bss.bss_eval_sources(refs, ests, compute_permutation=compute_permutation)
    return tuple(o.cpu().numpy() for o in out)
