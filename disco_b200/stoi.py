"""Classic STOI on the device: pystoi.stoi.stoi(x, y, fs_sig) (pystoi 0.3; Taal et al. 2011), batched, in float64.

A signal at another rate than 10 kHz is first resampled with Octave's resample() filter, as pystoi's resample_oct
does: a Kaiser-windowed sinc designed here on the host and applied by scipy.signal.resample_poly's polyphase scheme
(ops.resample_poly, csrc/stoi.cu).  The silent-frame removal, the 512-point float64 STFT, the one-third octave bands
and the clipped segment correlations then run in the kernels of ops.stoi.  Where fewer than 30 STFT frames remain
after the silent frames are removed, the score is 1e-5 and a RuntimeWarning is issued, as pystoi does.

Time is the last axis; every leading axis is a batch axis.  Inputs are float32 CUDA tensors.
"""
import warnings

import numpy as np
import torch

from . import ops

FS = 10000           # STOI's internal rate
N_FRAME = 256
NFFT = 512
NUM_BANDS = 15
MIN_FREQ = 150
N_SEG = 30           # STFT frames per segment: fewer frames score 1e-5


def resample_window(p, q):
    """Octave's resample() anti-aliasing filter for the rate change p / q (what pystoi's _resample_window_oct
    computes): 60 dB rejection, cutoff 1 / (2 max(p, q)) after reducing p / q, roll-off a tenth of the cutoff."""
    g = np.gcd(p, q)
    if g > 1:
        p /= g
        q /= g
    cutoff = 1. / (2 * max(p, q))
    roll_off = cutoff / 10
    rejection_db = 60.0
    L = np.ceil((rejection_db - 8) / (28.714 * roll_off))
    t = np.arange(-L, L + 1)
    ideal = 2 * p * cutoff * np.sinc(2 * cutoff * t)
    return np.kaiser(2 * L + 1, 0.1102 * (rejection_db - 8.7)) * ideal


def resample_taps(fs):
    """(taps, up, down) that bring fs to 10 kHz: the filter normalised to unit sum, as scipy's resample_poly takes it."""
    h = resample_window(FS, fs)
    g = int(np.gcd(FS, int(fs)))
    return h / np.sum(h), FS // g, int(fs) // g


def band_edges():
    """[(a_i, b_i)] of the 15 one-third octave bands from 150 Hz: band i sums the STFT bins a_i <= k < b_i, each edge
    the first bin nearest to 150 * 2^((2 i -+ 1) / 6) Hz (bin k at k * 10000 / 512 Hz).  csrc/stoi.cu holds the
    same table."""
    f = np.linspace(0, FS, NFFT + 1)[:NFFT // 2 + 1]
    k = np.arange(NUM_BANDS).astype(float)
    lo = MIN_FREQ * np.power(2., (2 * k - 1) / 6)
    hi = MIN_FREQ * np.power(2., (2 * k + 1) / 6)
    return [(int(np.argmin(np.square(f - a))), int(np.argmin(np.square(f - b)))) for a, b in zip(lo, hi)]


def to_10k(x, fs, lengths=None):
    """x [..., L] float32 CUDA tensor at fs -> float64 at 10 kHz (pystoi's resample_oct).  lengths (per row, or None):
    each row is resampled as its first lengths[s] samples, zero after ceil(lengths[s] 10000 / fs)."""
    if int(fs) != fs or fs < 1:
        raise ValueError("fs must be a positive integer rate, got %r" % (fs,))
    if int(fs) == FS:
        return x.double()
    taps, up, down = resample_taps(int(fs))
    return ops.resample_poly(x, torch.from_numpy(taps).to(x.device), up, down, lengths=lengths)


def length_10k(n, fs):
    """Samples at 10 kHz of n samples at fs: ceil(n up / down), resample_poly's output length."""
    if int(fs) == FS:
        return np.asarray(n)
    _, up, down = resample_taps(int(fs))
    return -(-np.asarray(n, dtype=np.int64) * up // down)


def _check(t, name):
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise TypeError("%s must be a CUDA tensor (disco_b200 has no CPU path)" % name)
    if t.dtype != torch.float32:
        raise TypeError("%s must be float32, got %s" % (name, t.dtype))


def _warn_if_short(n_frames):
    if bool((n_frames < N_SEG).any()):
        warnings.warn("Not enough STFT frames to compute intermediate intelligibility measure after removing silent "
                      "frames. Returning 1e-5. Please check you wav files", RuntimeWarning, stacklevel=3)


def stoi_pairs(cleans, degraded, pairs, fs, lengths=None):
    """STOI of (clean, degraded) pairs.  cleans [C, L], degraded [D, L] float32 CUDA tensors at rate fs, pairs [P, 2]
    integer (clean index, degraded index) -> d [P] float64.  Every signal is resampled once, and every clean's
    selection and band envelopes are computed once however many pairs share it.
    lengths [C] (integers, or None): clean c and every degraded signal paired with it are their first lengths[c]
    samples; a pair scores as pystoi on the two trimmed signals.  A degraded signal paired with cleans of different
    lengths raises ValueError."""
    _check(cleans, "cleans")
    _check(degraded, "degraded")
    if cleans.dim() != 2 or degraded.dim() != 2 or cleans.shape[1] != degraded.shape[1]:
        raise ValueError("cleans [C, L] / degraded [D, L] shape mismatch: %s / %s"
                         % (tuple(cleans.shape), tuple(degraded.shape)))
    pairs = torch.as_tensor(pairs).to(device=cleans.device, dtype=torch.int32).reshape(-1, 2).contiguous()
    if lengths is None:
        xc, xd = to_10k(cleans.contiguous(), fs), to_10k(degraded.contiguous(), fs)
        l10 = None
    else:
        C, D, L = cleans.shape[0], degraded.shape[0], cleans.shape[1]
        lc = ops.signal_lengths(lengths, (C,), L)
        pr = pairs.cpu().numpy().astype(np.int64)
        if pr.size and (pr[:, 0].min() < 0 or pr[:, 0].max() >= C or pr[:, 1].min() < 0 or pr[:, 1].max() >= D):
            raise IndexError("stoi: pair indices out of range (%d cleans, %d degraded signals)" % (C, D))
        ld = np.full(D, L, dtype=np.int32)
        ld[pr[:, 1]] = lc[pr[:, 0]]
        if np.any(ld[pr[:, 1]] != lc[pr[:, 0]]):
            raise ValueError("stoi: a degraded signal is paired with cleans of different lengths")
        xc, xd = to_10k(cleans.contiguous(), fs, lc), to_10k(degraded.contiguous(), fs, ld)
        l10 = length_10k(lc, fs)
        if int(l10.min()) < N_FRAME:
            raise ValueError("stoi: %d samples at 10 kHz; at least %d are needed" % (int(l10.min()), N_FRAME))
    if xc.shape[-1] < N_FRAME:
        raise ValueError("stoi: %d samples at 10 kHz; at least %d are needed" % (xc.shape[-1], N_FRAME))
    d, _, n_frames = ops.stoi(xc, xd, pairs, lengths=l10)
    _warn_if_short(n_frames)
    return d


def stoi(x, y, fs):
    """pystoi.stoi.stoi(x, y, fs) batched: x clean, y degraded, [..., L] float32 CUDA tensors of the same shape ->
    [...] float64 on the device."""
    _check(x, "x")
    _check(y, "y")
    if x.shape != y.shape:
        raise ValueError("x and y should have the same shape, found %s and %s" % (tuple(x.shape), tuple(y.shape)))
    lead, L = tuple(x.shape[:-1]), x.shape[-1]
    n = int(np.prod(lead, dtype=np.int64))
    idx = torch.arange(n, dtype=torch.int32, device=x.device)
    d = stoi_pairs(x.reshape(n, L), y.reshape(n, L), torch.stack((idx, idx), dim=1), fs)
    return d.reshape(lead)
