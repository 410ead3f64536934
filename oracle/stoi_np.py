"""Float64 NumPy restatement of classic STOI (pystoi 0.3, ``pystoi.stoi.stoi(x, y, fs_sig)``; Taal et al. 2011), the
score the reference's tango.main computes six times per node (tango.py:569-578).  pystoi is absent here, so parity
with it is unpinned; the resampler stage calls scipy's resample_poly, which is installed, and is pinned to it.

Two forms of steps 2-5 are kept: `stoi_10k` follows pystoi's vectorised code, `stoi_loop` materialises the
overlap-added signals and loops over frames, segments and bands one value at a time.  The tests require them to agree
to 1e-12."""
import warnings

import numpy as np
from scipy.signal import resample_poly

FS = 10000          # STOI's internal sample rate
N_FRAME = 256       # window / frame length
NFFT = 512
NUMBAND = 15
MINFREQ = 150
N = 30              # frames per intermediate intelligibility segment
BETA = -15.0        # lower SDR bound of the clipping
DYN_RANGE = 40      # dB below the loudest frame that a frame must reach to be kept
EPS = np.finfo(float).eps


def resample_window_oct(p, q):
    """pystoi.utils._resample_window_oct: Octave's resample() filter for the rate change p / q."""
    gcd = np.gcd(p, q)
    if gcd > 1:
        p /= gcd
        q /= gcd
    log10_rejection = -3.0
    stopband_cutoff_f = 1. / (2 * max(p, q))
    roll_off_width = stopband_cutoff_f / 10
    rejection_db = -20 * log10_rejection
    L = np.ceil((rejection_db - 8) / (28.714 * roll_off_width))
    t = np.arange(-L, L + 1)
    ideal_filter = 2 * p * stopband_cutoff_f * np.sinc(2 * stopband_cutoff_f * t)
    if 21 <= rejection_db <= 50:
        beta = 0.5842 * (rejection_db - 21) ** 0.4 + 0.07886 * (rejection_db - 21)
    elif rejection_db > 50:
        beta = 0.1102 * (rejection_db - 8.7)
    else:
        beta = 0.0
    return np.kaiser(2 * L + 1, beta) * ideal_filter


def resample_oct(x, p, q):
    """pystoi.utils.resample_oct: x at rate q -> rate p."""
    h = resample_window_oct(p, q)
    return resample_poly(x, p, q, window=h / np.sum(h))


def thirdoct(fs=FS, nfft=NFFT, num_bands=NUMBAND, min_freq=MINFREQ):
    """pystoi.utils.thirdoct: the one-third octave band matrix [num_bands, nfft/2 + 1] and the centre frequencies."""
    f = np.linspace(0, fs, nfft + 1)
    f = f[:int(nfft / 2) + 1]
    k = np.array(range(num_bands)).astype(float)
    cf = np.power(2. ** (1. / 3), k) * min_freq
    freq_low = min_freq * np.power(2., (2 * k - 1) / 6)
    freq_high = min_freq * np.power(2., (2 * k + 1) / 6)
    obm = np.zeros((num_bands, len(f)))
    for i in range(len(cf)):
        fl_ii = np.argmin(np.square(f - freq_low[i]))
        fh_ii = np.argmin(np.square(f - freq_high[i]))
        obm[i, fl_ii:fh_ii] = 1
    return obm, cf


def band_edges():
    """[(a_i, b_i)]: band i sums bins a_i <= k < b_i."""
    obm, _ = thirdoct()
    return [(int(np.flatnonzero(r)[0]), int(np.flatnonzero(r)[-1]) + 1) for r in obm]


OBM, _ = thirdoct()


def hann():
    return np.hanning(N_FRAME + 2)[1:-1]


def frame_energies(x):
    """20 log10(‖w x_i‖ + EPS) of the frames starting at 0, 128, ... (pystoi.utils.remove_silent_frames)."""
    w = hann()
    frames = np.array([w * x[i:i + N_FRAME] for i in range(0, len(x) - N_FRAME + 1, N_FRAME // 2)])
    return 20 * np.log10(np.linalg.norm(frames, axis=1) + EPS)


def selection(x):
    """Indices of the frames of x that remove_silent_frames keeps (raises ValueError below 256 samples)."""
    e = frame_energies(x)
    return np.flatnonzero((np.max(e) - DYN_RANGE - e) < 0)


def _overlap_and_add(frames, hop):
    num_frames, framelen = frames.shape
    segments = -(-framelen // hop)
    signal = np.pad(frames, ((0, segments), (0, segments * hop - framelen)))
    signal = signal.reshape((num_frames + segments, segments, hop))
    signal = np.transpose(signal, (1, 0, 2))
    signal = signal.reshape((-1, hop))
    signal = signal[:-segments]
    signal = signal.reshape((segments, num_frames + segments - 1, hop))
    signal = np.sum(signal, axis=0)
    end = (len(frames) - 1) * hop + framelen
    return signal.reshape(-1)[:end]


def remove_silent_frames(x, y, dyn_range=DYN_RANGE, framelen=N_FRAME, hop=N_FRAME // 2):
    """pystoi.utils.remove_silent_frames: the frames of x within dyn_range dB of its loudest, overlap-added (and the
    same frames of y)."""
    w = np.hanning(framelen + 2)[1:-1]
    x_frames = np.array([w * x[i:i + framelen] for i in range(0, len(x) - framelen + 1, hop)])
    y_frames = np.array([w * y[i:i + framelen] for i in range(0, len(x) - framelen + 1, hop)])
    x_energies = 20 * np.log10(np.linalg.norm(x_frames, axis=1) + EPS)
    mask = (np.max(x_energies) - dyn_range - x_energies) < 0
    return _overlap_and_add(x_frames[mask], hop), _overlap_and_add(y_frames[mask], hop)


def stft(x, win_size=N_FRAME, fft_size=NFFT, overlap=2):
    """pystoi.utils.stft: the last full frame is not taken (range(0, len - win, hop))."""
    hop = int(win_size / overlap)
    w = np.hanning(win_size + 2)[1:-1]
    return np.array([np.fft.rfft(w * x[i:i + win_size], n=fft_size) for i in range(0, len(x) - win_size, hop)])


def _too_few():
    warnings.warn("Not enough STFT frames to compute intermediate intelligibility measure after removing silent "
                  "frames. Returning 1e-5. Please check you wav files", RuntimeWarning)
    return 1e-5


def tob(x, y):
    """One-third octave band envelopes [15, n_frames] of x and y after the silent-frame removal."""
    x, y = remove_silent_frames(x, y)
    x_spec, y_spec = stft(x).transpose(), stft(y).transpose()
    return np.sqrt(np.matmul(OBM, np.square(np.abs(x_spec)))), np.sqrt(np.matmul(OBM, np.square(np.abs(y_spec))))


def stoi_10k(x, y):
    """Steps 2-5 of pystoi.stoi.stoi on 10 kHz float64 signals, vectorised as pystoi writes them."""
    x_tob, y_tob = tob(x, y)
    if x_tob.shape[-1] < N:
        return _too_few()
    x_segments = np.array([x_tob[:, m - N:m] for m in range(N, x_tob.shape[1] + 1)])
    y_segments = np.array([y_tob[:, m - N:m] for m in range(N, x_tob.shape[1] + 1)])
    norm_const = np.linalg.norm(x_segments, axis=2, keepdims=True) / (
        np.linalg.norm(y_segments, axis=2, keepdims=True) + EPS)
    y_segments_normalized = y_segments * norm_const
    clip_value = 10 ** (-BETA / 20)
    y_primes = np.minimum(y_segments_normalized, x_segments * (1 + clip_value))
    y_primes = y_primes - np.mean(y_primes, axis=2, keepdims=True)
    x_segments = x_segments - np.mean(x_segments, axis=2, keepdims=True)
    y_primes /= (np.linalg.norm(y_primes, axis=2, keepdims=True) + EPS)
    x_segments /= (np.linalg.norm(x_segments, axis=2, keepdims=True) + EPS)
    J, M = x_segments.shape[0], x_segments.shape[1]
    return np.sum(y_primes * x_segments) / (J * M)


def stoi_loop(x, y):
    """stoi_10k written out: the kept frames overlap-added sample by sample, one DFT bin sum per band and frame, one
    segment and band at a time."""
    w = hann()
    hop = N_FRAME // 2
    keep = selection(x)
    n_sel = len(keep)
    out_len = (n_sel - 1) * hop + N_FRAME
    xs, ys = np.zeros(out_len), np.zeros(out_len)
    for j, f in enumerate(keep):
        for r in range(N_FRAME):
            xs[j * hop + r] += w[r] * x[f * hop + r]
            ys[j * hop + r] += w[r] * y[f * hop + r]
    n_frames = len(range(0, out_len - N_FRAME, hop))
    if n_frames < N:
        return _too_few()
    edges = band_edges()
    X = np.zeros((NUMBAND, n_frames))
    Y = np.zeros((NUMBAND, n_frames))
    for t in range(n_frames):
        fx = np.fft.rfft(w * xs[t * hop:t * hop + N_FRAME], NFFT)
        fy = np.fft.rfft(w * ys[t * hop:t * hop + N_FRAME], NFFT)
        for i, (a, b) in enumerate(edges):
            X[i, t] = np.sqrt(sum(abs(fx[k]) ** 2 for k in range(a, b)))
            Y[i, t] = np.sqrt(sum(abs(fy[k]) ** 2 for k in range(a, b)))
    J = n_frames - N + 1
    total = 0.0
    for m in range(J):
        for i in range(NUMBAND):
            xv, yv = X[i, m:m + N], Y[i, m:m + N]
            alpha = np.sqrt(np.sum(xv ** 2)) / (np.sqrt(np.sum(yv ** 2)) + EPS)
            yp = np.minimum(alpha * yv, xv * (1 + 10 ** (-BETA / 20)))
            xc, yc = xv - xv.mean(), yp - yp.mean()
            xc = xc / (np.sqrt(np.sum(xc ** 2)) + EPS)
            yc = yc / (np.sqrt(np.sum(yc ** 2)) + EPS)
            total += np.sum(xc * yc)
    return total / (J * NUMBAND)


def to_10k(x, fs_sig):
    x = np.asarray(x, dtype=np.float64) if fs_sig == FS else resample_oct(np.asarray(x), FS, fs_sig)
    return x


def stoi(x, y, fs_sig):
    """pystoi.stoi.stoi(x, y, fs_sig) (classic STOI): x clean, y degraded, 1-D, same length."""
    if x.shape != y.shape:
        raise Exception("x and y should have the same length, found {} and {}".format(x.shape, y.shape))
    return stoi_10k(to_10k(x, fs_sig), to_10k(y, fs_sig))


def n_stft_frames(x10k):
    """STFT frames STOI scores for a 10 kHz clean: one less than the kept frames."""
    return len(selection(x10k)) - 1
