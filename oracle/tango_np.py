"""Loop-faithful NumPy/SciPy restatement of the reference's two-step distributed MWF
("Tango") — TEST INFRASTRUCTURE, see oracle/__init__.py.

Every function cites the reference lines (relative to /root/reference/) it follows and
keeps the reference's dtype flow (SURVEY.md App. A.5): complex64 STFTs, float32 oracle
masks, complex64 outer products averaged in complex64, single-precision generalised
eigen-solve (scipy.linalg.eig on complex64 -> LAPACK cggev), complex128 filters,
complex128 inner products rounded into complex64 outputs.

The per-(bin, frame) granularity of the reference (one np.outer / np.inner call per
time-frequency point) is kept in ``granularity='frame'`` because that is what makes
the reference's CPU path what it is; ``granularity='bin'`` evaluates the same sums
with one contraction per bin (same math and dtypes, different summation order).

Pinned by tests/test_oracle.py against tests/golden/*.npz, which hold outputs of the
reference's own offline_tango / intern_filter run through oracle/ref_shim.py.
"""
import sys

import numpy as np
import scipy.linalg

from oracle import librosa_np

EPS = sys.float_info.epsilon      # internal_formulas.py:6
ETA = 1e6                         # internal_formulas.py:7


# --------------------------------------------------------------------------- masks
def tf_mask(s, n, type="irm1", bin_thr=0):
    """dnn/utils.py:44-71 (twin: sigproc_utils.py:58-86)."""
    power = int(type[-1])
    if "irm" in type:
        xi = (abs(s) / np.maximum(abs(n), EPS)) ** power
        return xi / (1 + xi)
    if "ibm" in type:
        xi = (abs(s) / np.maximum(abs(n), EPS)) ** power
        return xi >= 10 ** (bin_thr / 10)          # math_utils.db2lin
    if "iam" in type:
        return (abs(s) / abs(s + n)) ** power
    raise ValueError('Unknown mask type. Should be "irmX", "ibmX" or "iamX"')


def vad_oracle_batch(x_, win_len=512, win_hop=256, thr=0.001, rat=2):
    """sigproc_utils.py:12-55: energy VAD, one decision per window, returned per sample."""
    x = x_ - np.mean(x_)
    x2 = abs(x ** 2)
    thr_ = thr * np.quantile(x2, 0.99)
    vad = np.zeros(len(x2))
    n_win = int(np.ceil((len(x2) - win_len) / win_hop + 1))
    for i in range(n_win):
        a, b = i * win_hop, min(i * win_hop + win_len, len(x2))
        seg = x2[a:b]
        if int(np.sum(seg > thr_)) >= int(len(seg) / rat):
            vad[a:b] = 1
    return vad


def get_mask(ss, sn, mask_type="irm1", ts=None, n_fft=512, n_hop=256):
    """tango.py:189-225, oracle branches only (no DNN in the oracle)."""
    if mask_type[:-1] in ("irm", "ibm", "iam"):
        return tf_mask(ss, sn, type=mask_type)
    if mask_type == "ivad":
        m = np.zeros(np.shape(ss))
        vad = vad_oracle_batch(ts, win_len=n_fft, win_hop=n_hop)[::n_hop]
        m[:, :len(vad)] = np.tile(vad, (np.shape(ss)[0], 1))
        return m
    raise ValueError("Unknown value for `mask_type`")


# --------------------------------------------------------------------------- filters
def intern_filter(Rxx, Rnn, mu=1, type="r1-mwf", rank="Full"):
    """internal_formulas.py:31-81.  Returns (W, (t1, sort_index))."""
    dim = np.shape(Rxx)[0]
    t1 = np.zeros(dim)
    t1[0] = 1.0                                            # :43  e1 selector
    order = None
    if type == "r1-mwf":                                   # :45-54
        vals, vecs = np.linalg.eig(Rxx)
        vals = np.real(vals)
        top = vals.argmax()
        R1 = np.outer(np.abs(vals[top]) * vecs[:, top], np.conjugate(vecs[:, top]).T)
        P = np.linalg.lstsq(Rnn, R1, rcond=None)[0]
        W = 1 / (mu + np.trace(P)) * P[:, 0]
    elif type == "gevd":                                   # :56-73
        vals, Q = scipy.linalg.eig(Rxx, Rnn)
        vals = np.maximum(vals, EPS * np.ones(vals.shape))
        vals = np.minimum(vals, ETA * np.ones(vals.shape))
        order = np.argsort(vals)
        Dm = np.diag(vals[order[::-1]])
        Q = Q[:, order[::-1]]
        if rank != "full":
            Dm[rank:, :] = 0
        gain = np.matmul(Dm, np.linalg.inv(Dm + mu * np.eye(dim)))
        W = np.matmul(Q, np.matmul(gain, np.linalg.inv(Q)))[:, 0]
        t1 = Q[:, 0] * np.linalg.inv(Q)[0, 0]
    elif type == "mwf":                                    # :74-76
        W = np.linalg.lstsq(Rnn + Rxx, Rxx, rcond=None)[0][:, 0]
    else:
        raise AttributeError("Unknown filter reference")
    return W, (t1, order)


def spatial_correlation_matrix(Rxx, x, lambda_cor=0.95, M=None):
    """internal_formulas.py:84-103: one step of the exponentially smoothed SCM."""
    upd = (1 - lambda_cor) * np.outer(x, np.conjugate(x).T)
    if M is not None:
        upd = M * upd
    return lambda_cor * Rxx + upd


# --------------------------------------------------------------------------- SCM / apply
def scm_bin(sig_f, granularity="frame"):
    """tango.py:357-364 / :433-440 for one frequency bin: mean_t a_t a_t^H, sig_f (D, T)."""
    if granularity == "frame":
        per_frame = [np.outer(sig_f[:, t], np.conjugate(sig_f[:, t]).T)
                     for t in range(sig_f.shape[1])]
        return np.mean(np.array(per_frame), axis=0)
    acc = np.einsum("it,jt->ij", sig_f, np.conjugate(sig_f))
    return (acc / sig_f.shape[1]).astype(sig_f.dtype)


def apply_bin(w, sig_f, conj=True, granularity="frame"):
    """tango.py:369-374 / :445-450: np.inner(conj(w), x[:, f, t]) for all t of one bin."""
    ww = np.conjugate(w) if conj else w
    if granularity == "frame":
        return np.array([np.inner(ww, sig_f[:, t]) for t in range(sig_f.shape[1])])
    return ww @ sig_f


def concatenate_signals(y, z, k, m=1):
    """tango.py:142-155: own mics, then m * z of nodes < k, then m * z of nodes > k."""
    z = np.array(z)
    return np.concatenate((y[k], m * z[:k], m * z[k + 1:]), axis=0)


# --------------------------------------------------------------------------- Tango
def offline_tango(y, s, n, vads=("irm1", "irm1"), mask_for_z="local", n_fft=512, n_hop=256,
                  mu=1, filter_type="gevd", rank=1, ref_mic=0, granularity="frame",
                  masks=None, double=False):
    """tango.py:252-457 with oracle masks (mods=None) and the reference microphone ref_mic of every node.

    ref_mic: the step-1 oracle mask is that of microphone ref_mic and applies to all the node's channels, and
    zn = Y[ref_mic] - z_y; the step-2 oracle mask is that of microphone 0.  The reference pins only ref_mic = 0
    (for any other value its tango.py:347 reads mask_z before node 0 has one); oracle/tango_f64.py states the same
    definition independently and tests/test_tango_routes_cpu.py holds the two together.
    y, s, n: [node][channel] 1-D float32 signals.  ``masks`` optionally overrides the
    oracle masks with externally supplied ones: (mask_z[K], mask_w[K]) of (F, T) arrays
    (what a DNN would deliver, tango.py:209-215).
    Returns the reference's 9 lists: yf, sf, nf, z_y, z_s, z_n, zn, masks_z, mask_w.
    Deployment mode (``s is None``: no clean components exist, masks must be given, mask_for_z='local'): the
    STFTs of s and n and the diagnostic outputs sf, nf, z_s, z_n -- which the reference only computes because
    its evaluation script has the clean signals -- are skipped (those lists come back as None).
    double=True evaluates the SAME algorithm in double precision (complex128 spectra, SCMs and LAPACK zggev):
    the float64 yardstick for the modes oracle/tango_f64.py does not restate (ragged arrays, 'compressed', ...).
    """
    K = len(y)
    F = n_fft // 2 + 1

    cdt = "complex128" if double else "complex64"

    def spec(x):
        if double:
            return librosa_np.stft(np.asarray(x, dtype=np.float64), n_fft=n_fft, hop_length=n_hop, center=True,
                                   dtype=np.complex128)
        return librosa_np.stft(np.asarray(x), n_fft=n_fft, hop_length=n_hop, center=True)

    Y = [np.array([spec(c) for c in y[k]]) for k in range(K)]              # :335
    deploy = s is None
    if deploy and (masks is None or mask_for_z != "local"):
        raise ValueError("deployment mode needs masks and mask_for_z='local'")
    S = None if deploy else [np.array([spec(c) for c in s[k]]) for k in range(K)]   # :336
    N = None if deploy else [np.array([spec(c) for c in n[k]]) for k in range(K)]   # :337
    T = Y[0].shape[-1]

    def two_outputs():
        return [np.zeros((F, T), cdt) for _ in range(K)]

    z_y, z_s, z_n = two_outputs(), two_outputs(), two_outputs()
    zn = [None] * K
    masks_z = [None] * K
    # ---- step 1: local filters, compressed signals (tango.py:326-376)
    for k in range(K):
        if masks is not None:
            mz = masks[0][k]
        else:
            mz = get_mask(S[k][ref_mic], N[k][ref_mic], vads[0], ts=np.asarray(s[k][ref_mic]),
                          n_fft=n_fft, n_hop=n_hop)                         # :338-342
        masks_z[k] = mz
        if mask_for_z is not None and "use_oracle_" in mask_for_z:          # :343-345
            s_hat, n_hat = S[k], N[k]
        else:
            s_hat = np.array([mz * ch for ch in Y[k]])                      # :347
            n_hat = np.array([(1 - mz) * ch for ch in Y[k]])                # :348
        for f in range(F):
            Rss = scm_bin(s_hat[:, f, :], granularity)                      # :357-363
            Rnn = scm_bin(n_hat[:, f, :], granularity)                      # :364
            w, _ = intern_filter(Rss, Rnn, mu=mu, type=filter_type, rank=rank)   # :367
            z_y[k][f] = apply_bin(w, Y[k][:, f, :], True, granularity)      # :370
            if not deploy:
                z_s[k][f] = apply_bin(w, S[k][:, f, :], True, granularity)  # :371
                z_n[k][f] = apply_bin(w, N[k][:, f, :], True, granularity)  # :372
        zn[k] = Y[k][ref_mic] - z_y[k]                                      # :376

    # ---- exchange + step-2 masks (tango.py:379-409)
    z_rs = [z.copy() for z in z_y]
    z_rn = [z.copy() for z in z_y]
    mask_w = [None] * K
    for k in range(K):
        if masks is not None:
            mask_w[k] = masks[1][k]
        else:
            mask_w[k] = get_mask(S[k][0], N[k][0], vads[1], ts=np.asarray(s[k][0]),
                                 n_fft=n_fft, n_hop=n_hop)                  # :391-394
        if mask_for_z == "distant":                                         # :396-398
            z_rs[k] = z_rs[k] * mask_w[k]
            z_rn[k] = z_rn[k] * (1 - mask_w[k])
        elif mask_for_z == "compressed":                                    # :399-403
            mc = get_mask(z_s[k], z_n[k], vads[0])
            z_rs[k] = z_rs[k] * mc
            z_rn[k] = z_rn[k] * (1 - mc)
        elif mask_for_z == "use_oracle_refs":                               # :404-406
            z_rs[k], z_rn[k] = S[k][ref_mic], N[k][ref_mic]
        elif mask_for_z == "use_oracle_zs":                                 # :407-409
            z_rs[k], z_rn[k] = z_s[k], z_n[k]

    # ---- step 2: global filters (tango.py:411-450)
    yf, sf, nf = two_outputs(), two_outputs(), two_outputs()
    for k in range(K):
        s_hat_w = [np.array([mask_w[j] * ch for ch in Y[j]]) for j in range(K)]      # :413
        n_hat_w = [np.array([(1 - mask_w[j]) * ch for ch in Y[j]]) for j in range(K)]  # :414
        ms, mn = 1, 1
        if mask_for_z == "local":                                           # :416-418
            ms, mn = mask_w[k], 1 - mask_w[k]
        elif mask_for_z is None:                                            # :419-422
            z_rn = zn
        elif mask_for_z == "use_oracle_sigs":
            raise NotImplementedError("'use_oracle_sigs' indexes z by node with per-channel "
                                      "arrays in the reference (tango.py:423-427); not restated")
        phi_s_in = concatenate_signals(s_hat_w, z_rs, k, ms)               # :431
        phi_n_in = concatenate_signals(n_hat_w, z_rn, k, mn)               # :432
        in_y = concatenate_signals(Y, z_y, k)                              # :382
        if not deploy:
            in_s = concatenate_signals(S, z_s, k)                          # :383
            in_n = concatenate_signals(N, z_n, k)                          # :384
        for f in range(F):
            Rss = scm_bin(phi_s_in[:, f, :], granularity)                   # :433-439
            Rnn = scm_bin(phi_n_in[:, f, :], granularity)                   # :440
            w, _ = intern_filter(Rss, Rnn, mu=mu, type=filter_type, rank=rank)   # :443
            yf[k][f] = apply_bin(w, in_y[:, f, :], True, granularity)       # :446
            if not deploy:
                sf[k][f] = apply_bin(w, in_s[:, f, :], True, granularity)   # :447
                nf[k][f] = apply_bin(w, in_n[:, f, :], True, granularity)   # :448
    if deploy:
        sf = nf = z_s = z_n = None
    return yf, sf, nf, z_y, z_s, z_n, zn, masks_z, mask_w
