"""The step right after the beamformer (SURVEY.md §8 f-2): back to the time domain and scoring, on
the device.  Mirrors the post-processing of disco_theque/speech_enhancement/tango.py:526-539 (six
``lb.core.istft`` calls per node) and disco_theque/metrics.py (``si_sdr`` :342-391, ``snr`` helpers).

`to_time` runs ONE batched iSTFT kernel launch for all outputs, nodes and utterances.  `fw_snr` / `fw_sd`
(metrics.py:63-128, 211-279) run the whole third-octave Butterworth bank over all signals in one launch of
the IIR filter-bank kernel (csrc/filterbank.cu) that returns only the band powers; the band weighting is a
few float64 operations on [..., 17] tensors.  `si_sdr`, `snr`, `sd` are float64 reductions (torch on the
device).  BSS-eval's SDR / SIR / SAR (mir_eval.separation.bss_eval_sources) run on the float64 projection kernels of
csrc/bss.cu (disco_b200/bss_eval.py) and STOI (pystoi.stoi.stoi) on the float64 kernels of csrc/stoi.cu
(disco_b200/stoi.py); `tango_scores` is the whole scoring block of tango.main, STOI included on request.

All metrics are batched: TIME IS THE LAST AXIS, every leading axis is a batch axis (the reference's
functions take one 1-D signal per call).
"""
import math

import numpy as np
import torch

from . import ops

# band importance function of the reference (metrics.py:81-95): ANSI S3.5 third-octave weights
_I_WIDE = np.array([83, 95, 150, 289, 440, 578, 653, 711, 818, 844, 882, 898, 868, 844, 771, 527, 364, 185]) * 1e-4
_F_WIDE = np.array([160, 200, 250, 315, 400, 500, 630, 800, 1000, 1250, 1600, 2000, 2500, 3150, 4000, 5000, 6300, 8000])
_I_NARROW = np.array([128, 320, 320, 447, 447, 639, 639, 767, 959, 1182, 1214, 1086, 1086, 757]) * 1e-4
_F_NARROW = np.array([200, 250, 315, 400, 500, 630, 800, 1000, 1250, 1600, 2000, 2500, 3150, 4000])
_G_OCTAVE = 10.0 ** 0.3          # IEC 61260-1:2014 octave ratio (what acoustics.signal.OctaveBand implements)


def to_time(outputs, length, n_fft=512, names=("yf", "z_y", "sf", "nf", "z_s", "z_n"), layout="FT", lengths=None):
    """outputs: dict from tango_batched ([B, K, F, T] for layout 'FT', [B, K, T, F] for 'TF').
    Returns {name: [B, K, length] float32} for the names present (tango.py:526-539).
    lengths [B] (the tango_batched argument): utterance b is the iSTFT of its frames [0, 1 + lengths[b] // hop) to
    lengths[b] samples, zero after them (ops.istft_lengths); None: every utterance is `length` samples long."""
    present = [n for n in names if n in outputs]
    if not present:
        return {}
    specs = []
    for n in present:
        S = outputs[n]
        specs.append(ops.transpose_last2(S.contiguous()) if layout == "FT" else S)
    stack = torch.stack(specs).contiguous()                    # [n, B, K, T, F]
    if lengths is None:
        x = ops.istft(stack, int(length), n_fft)               # [n, B, K, length]
    else:
        per_utt = ops.signal_lengths(lengths, stack.shape[1:2], int(length))
        x = ops.istft_lengths(stack, np.broadcast_to(per_utt, (len(present),) + per_utt.shape), int(length), n_fft)
    return {n: x[i] for i, n in enumerate(present)}


def si_sdr(reference, estimation):
    """Scale-invariant SDR in dB over the last axis (metrics.py:342-391), float64 on the device."""
    ref = torch.as_tensor(reference).to(torch.float64)
    est = torch.as_tensor(estimation).to(device=ref.device, dtype=torch.float64)
    est, ref = torch.broadcast_tensors(est, ref)
    energy = (ref * ref).sum(-1, keepdim=True)
    proj = ((ref * est).sum(-1, keepdim=True) / energy) * ref
    noise = est - proj
    return 10.0 * torch.log10((proj * proj).sum(-1) / (noise * noise).sum(-1))


def snr_db(signal, noise):
    """10 log10 of the power ratio over the last axis (the plain SNR used around tango.py:552-593)."""
    s = torch.as_tensor(signal).to(torch.float64)
    n = torch.as_tensor(noise).to(device=s.device, dtype=torch.float64)
    return 10.0 * torch.log10((s * s).sum(-1) / (n * n).sum(-1))


# ------------------------------------------------------------------ frequency-weighted metrics
def third_octave_bands(fs):
    """Centre frequencies and importance weights the reference uses at sampling rate fs (metrics.py:80-95):
    the bands whose upper edge F * 2**(1/6) lies below fs / 2."""
    F, I = (_F_WIDE, _I_WIDE) if fs / 2 > 4500 else (_F_NARROW, _I_NARROW)
    n = int(np.sum(F * 2 ** (1 / 6) < fs / 2))
    return F[:n], I[:n]


def _butter_bandpass(order, lo, hi):
    """Digital Butterworth band-pass of prototype order `order` (filter order 2 * order), edges normalised to
    Nyquist = 1: analog prototype -> pre-warped band-pass transform -> bilinear transform -> polynomials
    (the textbook route, the one scipy.signal.butter(order, [lo, hi], 'bandpass') follows)."""
    fs = 2.0
    w = 2 * fs * np.tan(np.pi * np.array([lo, hi], dtype=np.float64) / fs)
    bw, wo = w[1] - w[0], math.sqrt(w[0] * w[1])
    m = np.arange(-order + 1, order, 2)
    p_lp = -np.exp(1j * np.pi * m / (2 * order)) * bw / 2                  # Butterworth poles, scaled to bw
    root = np.sqrt(p_lp ** 2 - wo ** 2)
    p_bp = np.concatenate((p_lp + root, p_lp - root))
    z_bp = np.zeros(order)
    k_bp = bw ** order
    fs2 = 2 * fs
    z_d = np.append((fs2 + z_bp) / (fs2 - z_bp), -np.ones(len(p_bp) - len(z_bp)))
    p_d = (fs2 + p_bp) / (fs2 - p_bp)
    k_d = k_bp * np.real(np.prod(fs2 - z_bp) / np.prod(fs2 - p_bp))
    return np.real(k_d * np.poly(z_d)), np.real(np.poly(p_d))


def third_octave_filterbank(F, fs, order=8):
    """Reference signature (sigproc_utils.py:90-116): row i = coefficients (b, a) of the order-`order`
    Butterworth band-pass over the third-octave band around F[i].  Band edges: IEC 61260-1 base-10 exact
    mid-band frequency of the band nearest to F[i], times G**(-1/6), G**(+1/6), G = 10**0.3."""
    F = np.atleast_1d(np.asarray(F, dtype=np.float64))
    b = np.zeros((len(F), 2 * order + 1))
    a = np.zeros((len(F), 2 * order + 1))
    for i, f in enumerate(F):
        idx = np.round(3 * np.log(f / 1000.0) / np.log(_G_OCTAVE))
        centre = 1000.0 * _G_OCTAVE ** (idx / 3)
        lo, hi = centre * _G_OCTAVE ** (-1 / 6), centre * _G_OCTAVE ** (1 / 6)
        b[i], a[i] = _butter_bandpass(order, lo * 2 / fs, hi * 2 / fs)
    return b, a


_bank_cache = {}


def _bank(fs, order, device):
    key = (int(fs), int(order), str(device))
    if key not in _bank_cache:
        F, I = third_octave_bands(fs)
        b, a = third_octave_filterbank(F, fs, order=order)
        ba = torch.from_numpy(np.stack([b, a], axis=1)).to(device)          # [N, 2, 2*order+1]
        _bank_cache[key] = (F, torch.from_numpy(I / np.sum(I)).to(device), ba)
    return _bank_cache[key]


def band_powers_db(x, fs, order=4, vad=None):
    """10 log10 of the variance of every third-octave band of x ([..., L] float32 on the device) over the
    non-zero filter outputs, or over the samples with vad != 0 (metrics.py:96-107) -> [..., N] float64."""
    _, _, ba = _bank(fs, order, x.device)
    st = ops.band_stats(x, ba, sel=None if vad is None else vad.to(torch.float32))
    cnt, sm, sq = st[..., 0], st[..., 1], st[..., 2]
    mean = sm / cnt
    return 10.0 * torch.log10(sq / cnt - mean * mean)


def fw_snr(s, n, fs, vad_tar=None, vad_noi=None, clipping=1, db=True):
    """Frequency-weighted SNR (reference metrics.py:63-128), batched over the leading axes.
    Returns (fqwt_snr [..., N], fw_snr_mean [...], F)."""
    F, w, _ = _bank(fs, 4, s.device)
    snr_var = band_powers_db(s, fs, 4, vad_tar) - band_powers_db(n, fs, 4, vad_noi)
    if clipping:
        snr_var = snr_var.clamp(-15.0, 25.0)
    fq = w * snr_var
    mean = fq.sum(-1)
    if not db:
        fq, mean = 10.0 ** (fq / 10.0), 10.0 ** (mean / 10.0)
    return fq, mean, F


def fw_sd(s_out, s_in, fs, clipping=1, db=True, *, sel_out=None, sel_in=None):
    """Frequency-weighted speech distortion (reference metrics.py:211-279).  Returns (fqwt_sd, fw_sd_mean, F).
    sel_out / sel_in (like s_out, or None): band statistics of that signal over its samples with sel != 0 only (as
    fw_snr's vad_tar / vad_noi)."""
    F, w, _ = _bank(fs, 4, s_out.device)
    sd_var = band_powers_db(s_in, fs, 4, sel_in) - band_powers_db(s_out, fs, 4, sel_out)
    if clipping:
        sd_var = sd_var.clamp(0.0, 25.0)
    fq = w * sd_var
    mean = fq.sum(-1)
    if not db:
        fq, mean = 10.0 ** (fq / 10.0), 10.0 ** (mean / 10.0)
    return fq, mean, F


def _var_nonzero(x):
    x = x.to(torch.float64)
    nz = (x != 0)
    cnt = nz.sum(-1)
    mean = x.sum(-1) / cnt
    return ((x - mean.unsqueeze(-1)) ** 2 * nz).sum(-1) / cnt


def snr(s, n, db=True):
    """metrics.py:9-23: ratio of the variances of the non-zero samples."""
    r = _var_nonzero(s) / _var_nonzero(n)
    return 10.0 * torch.log10(r) if db else r


def delta_snr(s_out, n_out, s_in, n_in, db=True):
    """metrics.py:26-45."""
    d = snr(s_out, n_out, True) - snr(s_in, n_in, True)
    return d if db else 10.0 ** (d / 10.0)


def sd(s_out, s_in, db=True):
    """metrics.py:48-62."""
    r = _var_nonzero(s_in) / _var_nonzero(s_out)
    return 10.0 * torch.log10(r) if db else r


def tango_scores(y, s, n, s_dry, n_dry, times, fs, *, stoi=False, lengths=None):
    """The scoring block of the reference's tango.main (tango.py:541-593), batched over utterances and nodes.
    y, s, n [B, K, L]: mixture, target and noise at each node's reference microphone; s_dry, n_dry [B, L_dry] the dry
    sources of every utterance; times: the to_time() outputs ('yf', 'z_y', 'sf', 'nf', 'z_s', 'z_n', each [B, K, L]);
    float32 CUDA tensors.  Every signal is cut to [fs:min_len] as the reference does.
    Returns (results, resultsz) [B, K] float64 tensors keyed like the reference's two result pickles, without
    'snr_in_raw' (the caller's SNRs), and without 'delta_stoi*' unless stoi=True.

    bss(refs, ests) is only read at row 0, and row 0's scores depend on no other estimate row, so only the first row
    of each estimate set is correlated: (sh, szh, y) against the node's (s, n), and the same rows of all K nodes of an
    utterance against its dry (s_dry, n_dry), whose Gram matrix is factored once for the K nodes.

    stoi=True adds tango.py:569-578 under the reference's key names: results 'delta_stoi_cnv' = stoi(s, sh) -
    stoi(s, y) and 'delta_stoi_dry' = stoi(s_dry, sh) - stoi(s_dry, y); resultsz 'delta_stoi' and 'delta_stoi_dry',
    the same with szh.  The six calls of a node are six pairs of 2 cleans (s, and s_dry shared by the utterance's
    nodes) and 3 degraded signals (y, sh, szh): each signal is resampled once and each clean's silent-frame selection
    and band envelopes are computed once.

    lengths [B] (the tango_batched / to_time argument, or None): utterance b is scored over [fs, min(lengths[b],
    min_len)), as tango_scores scores that utterance alone, trimmed.  Every signal of the utterance is taken as zero
    after that.  BSS-eval and STOI see the zero-padded rows (trailing zeros change no projection norm; STOI's frame
    selection stops at each utterance's own last frame); fw_snr / fw_sd filter whole rows, which does not change the
    causal filter outputs before the end, and take their band statistics over the samples before it."""
    from . import bss_eval
    B, K, L = y.shape
    min_len = min(L, times["yf"].shape[-1], s_dry.shape[-1], n_dry.shape[-1])
    keep = None
    if lengths is None:
        cut = lambda x: x[..., fs:min_len]
    else:
        lb = np.minimum(ops.signal_lengths(lengths, (B,), L), min_len) - fs            # samples scored per utterance
        if int(lb.min()) < 1:
            raise ValueError("tango_scores: an utterance ends before the first second (fs samples) it skips")
        Ls = min_len - fs
        keep = torch.arange(Ls, device=y.device)[None, :] < torch.from_numpy(lb).to(y.device)[:, None]    # [B, Ls]
        tail = lambda x: (~keep).view((B,) + (1,) * (x.dim() - 2) + (Ls,))
        cut = lambda x: x[..., fs:min_len].masked_fill(tail(x), 0.0)
    sh, szh, yy = cut(times["yf"]), cut(times["z_y"]), cut(y)
    sf, nf, szf, nzf = cut(times["sf"]), cut(times["nf"]), cut(times["z_s"]), cut(times["z_n"])
    ss, nn, sd_, nd_ = cut(s), cut(n), cut(s_dry), cut(n_dry)
    rows = torch.stack((sh, szh, yy), dim=2)                                     # [B, K, 3, Ls]
    refs = torch.stack((ss, nn), dim=2)                                          # [B, K, 2, Ls]
    sdr, sir, sar = bss_eval.first_row_scores(refs.contiguous(), rows.contiguous())          # [B, K, 3]
    refs_dry = torch.stack((sd_, nd_), dim=1)                                    # [B, 2, Ls]
    d_sdr, d_sir, d_sar = bss_eval.first_row_scores(refs_dry.contiguous(),
                                                    rows.reshape(B, K * 3, -1).contiguous())
    d_sdr, d_sir, d_sar = (x.view(B, K, 3) for x in (d_sdr, d_sir, d_sar))

    # band statistics: without lengths over the non-zero filter outputs; with lengths over the samples that are both
    # before the utterance's end and non-zero outputs of the trimmed signal (the outputs are zero exactly up to the
    # first non-zero input sample: the band-passes have b0 != 0)
    own = (lambda x: None) if keep is None else (lambda x: _scored_samples(x, keep))
    sd_k = sd_.unsqueeze(1).expand(B, K, -1)
    _, snr_out, _ = fw_snr(sf, nf, fs, vad_tar=own(sf), vad_noi=own(nf))
    _, snr_in, _ = fw_snr(ss, nn, fs, vad_tar=own(ss), vad_noi=own(nn))
    _, snr_in_dry, _ = fw_snr(sd_, nd_, fs, vad_tar=own(sd_), vad_noi=own(nd_))
    _, snr_out_z, _ = fw_snr(szf, nzf, fs, vad_tar=own(szf), vad_noi=own(nzf))
    snr_in_dry = snr_in_dry.unsqueeze(1).expand(B, K)
    _, sd_cnv, _ = fw_sd(sf, ss, fs, sel_out=own(sf), sel_in=own(ss))
    _, sd_dry, _ = fw_sd(sf, sd_k, fs, sel_out=own(sf), sel_in=own(sd_k))
    _, sd_cnv_z, _ = fw_sd(szf, ss, fs, sel_out=own(szf), sel_in=own(ss))
    _, sd_dry_z, _ = fw_sd(szf, sd_k, fs, sel_out=own(szf), sel_in=own(sd_k))

    shared = {"snr_in_cnv": snr_in, "snr_in_dry": snr_in_dry,
              "sdr_in_cnv": sdr[..., 2], "sir_in_cnv": sir[..., 2],
              "sdr_in_dry": d_sdr[..., 2], "sir_in_dry": d_sir[..., 2], "sar_in_dry": d_sar[..., 2]}
    results = {"sar_cnv": sar[..., 0], "sir_cnv": sir[..., 0], "sdr_cnv": sdr[..., 0],
               "snr_out": snr_out, "fw_sd_cnv": sd_cnv, "fw_sd_dry": sd_dry,
               "sar_dry": d_sar[..., 0], "sir_dry": d_sir[..., 0], "sdr_dry": d_sdr[..., 0], **shared}
    resultsz = {"sar_cnv": sar[..., 1], "sir_cnv": sir[..., 1], "sdr_cnv": sdr[..., 1],
                "snr_out": snr_out_z, "fw_sd_cnv": sd_cnv_z, "fw_sd_dry": sd_dry_z,
                "sar_dry": d_sar[..., 1], "sir_dry": d_sir[..., 1], "sdr_dry": d_sdr[..., 1], **shared}
    if stoi:
        d = _tango_stoi(ss, sd_, yy, sh, szh, fs, None if keep is None else lb)  # [B, K, 6]
        results["delta_stoi_cnv"], results["delta_stoi_dry"] = d[..., 1] - d[..., 0], d[..., 4] - d[..., 3]
        resultsz["delta_stoi"], resultsz["delta_stoi_dry"] = d[..., 2] - d[..., 0], d[..., 5] - d[..., 3]
    return results, resultsz


def _scored_samples(x, keep):
    """float32 0/1 like x [B, ..., Ls]: samples n with first_b <= n and keep[b, n], first_b the first non-zero sample
    of the row (Ls for an all-zero row, which then selects nothing)."""
    nz = x != 0
    first = torch.where(nz.any(-1), nz.to(torch.int8).argmax(-1), x.shape[-1])
    n = torch.arange(x.shape[-1], device=x.device)
    k = keep.view((keep.shape[0],) + (1,) * (x.dim() - 2) + (keep.shape[1],))
    return ((n >= first.unsqueeze(-1)) & k).to(torch.float32)


def _tango_stoi(s, s_dry, y, sh, szh, fs, lengths=None):
    """STOI of the six pairs of every node, [B, K, 6]: (s, y), (s, sh), (s, szh), (s_dry, y), (s_dry, sh),
    (s_dry, szh).  s, y, sh, szh [B, K, L]; s_dry [B, L]; lengths [B] (host, or None): samples per utterance."""
    from . import stoi as _stoi
    B, K, L = s.shape
    cleans = torch.cat((s.reshape(B * K, L), s_dry.reshape(B, L)))               # node cleans, then dry cleans
    degraded = torch.stack((y, sh, szh), dim=2).reshape(B * K * 3, L)            # [B, K, 3] rows
    node = torch.arange(B * K, device=s.device)
    dry = B * K + node // K
    deg = 3 * node[:, None] + torch.arange(3, device=s.device)                   # [B K, 3]
    cl = torch.stack((node, dry), dim=1)[:, :, None].expand(B * K, 2, 3)         # [B K, 2, 3]
    pairs = torch.stack((cl, deg[:, None, :].expand(B * K, 2, 3)), dim=-1)       # [B K, 2, 3, 2]
    lc = None if lengths is None else np.concatenate((np.repeat(lengths, K), lengths))
    d = _stoi.stoi_pairs(cleans.contiguous(), degraded.contiguous(), pairs.reshape(-1, 2), fs, lengths=lc)
    return d.view(B, K, 6)
