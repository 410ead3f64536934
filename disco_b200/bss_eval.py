"""BSS-eval source scores on the device: mir_eval.separation.bss_eval_sources, batched, in float64.

For references r_1 .. r_n and an estimate e, mir_eval splits e into P_j e (target plus its filtering distortion), the
interference P_all e - P_j e and the artifacts e - P_all e, where P_S projects onto the references of S delayed by
0 .. flen-1 samples (flen = 512), and scores

    SDR = 10 log10(‖P_j e‖² / ‖e - P_j e‖²)
    SIR = 10 log10(‖P_j e‖² / ‖P_all e - P_j e‖²)
    SAR = 10 log10(‖P_all e‖² / ‖e - P_all e‖²)

with a zero (here: non-positive after rounding) denominator giving +inf.  The projections are orthogonal, so every
energy follows from ‖e‖² and the projection norms ops.bss_eval computes (csrc/bss.cu); the dB values and the
permutation search are a few float64 operations here.

Time is the last axis and every leading axis is a batch axis.  An estimate tensor with one axis more than the
references, [..., E, nsrc, L], holds E estimate sets scored against the same references: their Gram matrix is built
and factored once.
"""
import itertools

import torch

from . import ops


def _db(num, den):
    """10 log10(num / den), +inf where den <= 0 (mir_eval's _safe_db; rounding can leave a tiny negative energy)."""
    pos = den > 0
    val = 10.0 * torch.log10(num / torch.where(pos, den, torch.ones_like(den)))
    return torch.where(pos, val, torch.full_like(val, float("inf")))


def pair_scores(norms, nsrc):
    """Scores of every (estimate row, reference) pair from ops.bss_eval norms [..., R, 1 + 2 nsrc].
    Returns sdr, sir [..., R, nsrc] (row scored against reference k) and sar [..., R]."""
    ee = norms[..., 0]
    blocks = norms[..., 1:1 + nsrc]
    single = norms[..., 1 + nsrc:1 + 2 * nsrc]
    p_all = blocks.sum(-1)
    interf = p_all.unsqueeze(-1) - single
    # reference 0 leads the full factor: its interference is exactly the energy of the other blocks
    interf[..., 0] = blocks[..., 1:].sum(-1) if nsrc > 1 else torch.zeros_like(ee)
    sdr = _db(single, ee.unsqueeze(-1) - single)
    sir = _db(single, interf)
    sar = _db(p_all, ee - p_all)
    return sdr, sir, sar


def _check(refs, ests):
    for t, name in ((refs, "reference_sources"), (ests, "estimated_sources")):
        if not isinstance(t, torch.Tensor) or not t.is_cuda:
            raise TypeError("%s must be a CUDA tensor (disco_b200 has no CPU path)" % name)
        if t.dtype != torch.float32:
            raise TypeError("%s must be float32, got %s" % (name, t.dtype))


def bss_eval_sources(reference_sources, estimated_sources, compute_permutation=True, flen=512):
    """mir_eval.separation.bss_eval_sources over batches.
    reference_sources [..., nsrc, L]; estimated_sources [..., nsrc, L] or [..., E, nsrc, L], float32 CUDA tensors.
    Returns sdr, sir, sar [..., (E,) nsrc] float64 and perm [..., (E,) nsrc] int64 on the device.  With
    compute_permutation, every (estimate, reference) pair is scored and, per estimate set, the permutation with the
    largest mean SIR is chosen (the first on ties, as np.argmax); perm[i] is the estimate assigned to reference i and
    the scores are those of that assignment.  Without it, estimate j is scored against reference j."""
    refs, ests = reference_sources, estimated_sources
    _check(refs, ests)
    if refs.dim() < 2:
        raise ValueError("reference_sources must be [..., nsrc, L]")
    lead, (nsrc, L) = tuple(refs.shape[:-2]), tuple(refs.shape[-2:])
    if nsrc > 4:
        raise NotImplementedError("bss_eval_sources: at most 4 sources (got %d)" % nsrc)
    if ests.dim() == refs.dim():
        if ests.shape != refs.shape:
            raise ValueError("estimated_sources shape %s, expected %s" % (tuple(ests.shape), tuple(refs.shape)))
        E, extra = 1, ()
    elif ests.dim() == refs.dim() + 1 and tuple(ests.shape[:-3]) == lead and tuple(ests.shape[-2:]) == (nsrc, L):
        E, extra = ests.shape[-3], (ests.shape[-3],)
    else:
        raise ValueError("estimated_sources shape %s, expected %s or %s" % (
            tuple(ests.shape), tuple(refs.shape), lead + ("E", nsrc, L)))
    S = 1
    for d in lead:
        S *= d
    norms = ops.bss_eval(refs.reshape(S, nsrc, L).contiguous(), ests.reshape(S, E * nsrc, L).contiguous(), flen)
    sdr, sir, sar = pair_scores(norms.view(S, E, nsrc, 1 + 2 * nsrc), nsrc)    # [S, E, j (estimate), k (reference)]
    dev = norms.device
    if compute_permutation:
        perms = torch.tensor(list(itertools.permutations(range(nsrc))), dtype=torch.int64, device=dev)   # [P, nsrc]
        cols = torch.arange(nsrc, device=dev)
        mean_sir = sir[:, :, perms, cols].mean(-1)                                  # [S, E, P]
        perm = perms[mean_sir.argmax(-1)]                                          # [S, E, nsrc]
    else:
        perm = torch.arange(nsrc, device=dev).expand(S, E, nsrc)
    # score of reference i = that of the pair (estimate perm[i], reference i)
    si = torch.arange(S, device=dev)[:, None, None]
    ei = torch.arange(E, device=dev)[None, :, None]
    ri = torch.arange(nsrc, device=dev)[None, None, :]
    shape = lead + extra + (nsrc,)
    return (sdr[si, ei, perm, ri].reshape(shape), sir[si, ei, perm, ri].reshape(shape), sar[si, ei, perm].reshape(shape),
            perm.reshape(shape).contiguous())


def first_row_scores(references, first_rows, flen=512):
    """SDR, SIR, SAR of row 0 of estimate sets against reference 0, the only entries the reference's evaluation reads
    (tango.py:552-567 keeps bss(...)[k][0]).  Row 0's scores depend on no other estimate row, so only it is
    correlated: references [..., nsrc, L], first_rows [..., E, L] (row 0 of E estimate sets sharing the references)
    -> sdr, sir, sar [..., E] float64."""
    _check(references, first_rows)
    lead, (nsrc, L) = tuple(references.shape[:-2]), tuple(references.shape[-2:])
    if tuple(first_rows.shape[:-2]) != lead or first_rows.shape[-1] != L:
        raise ValueError("first_rows shape %s, expected %s" % (tuple(first_rows.shape), lead + ("E", L)))
    E = first_rows.shape[-2]
    S = 1
    for d in lead:
        S *= d
    norms = ops.bss_eval(references.reshape(S, nsrc, L).contiguous(), first_rows.reshape(S, E, L).contiguous(), flen)
    sdr, sir, sar = pair_scores(norms, nsrc)
    return (sdr[..., 0].reshape(lead + (E,)), sir[..., 0].reshape(lead + (E,)), sar.reshape(lead + (E,)))
