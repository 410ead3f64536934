"""Online Tango as a stream: push audio chunk by chunk, get the beamformed samples back about a frame later.

`online_tango` (online.py) runs the causal variant of Tango over a finished recording.  `OnlineTangoStream` runs the
same computation on audio as it arrives, and a causal mask estimator may compute the masks of each run of frames from
the frames just analysed (the step's own STFT and step-1 outputs).  Whatever the chunk sizes, the outputs equal
`online_tango` on the whole signal (with the masks the estimator returned) and `ops.istft` of its `yf`, value for
value: every stage is a deterministic kernel that works per frame or per block of frames, so the stream evaluates the
same operations in the same order, only at different times.

Per push, for every run of newly completed frames (a run never crosses a block boundary):
    stream_stft          the run's frames from the carried last n_fft samples and the chunk (csrc/stream.cu)
    filter_sum_blocks    step 1 (z, zn) and step 2 (yf) with the filters in force, W_(j - lag) for block j
    mask_fn              the run's masks, kept in the open block's buffers
    scm_recursive        once a block's last masks are in: its statistics from the carried matrices,
    mwf_solve            and the block's filters W1_j, W2_j
    stream_istft         the hop blocks of yf that became final (csrc/istft.cu)
"""
import numpy as np
import torch

from . import ops

N_FFTS = (256, 512, 1024)


def emission(length, n_fft=512, final=False):
    """What the stream has emitted after `length` samples: (frames out, time samples out).

    H = n_fft // 2.  Frame t reads samples [t H - H, t H + H) (librosa center=True, reflected at the start); it is out
    once every sample it reads has arrived: frame 0 at length >= H + 1, frame t >= 1 at length >= (t + 1) H, so frames
    0 .. length // H - 1 once length > H.  Hop block j of the output (samples [(j - 1) H, j H)) is final once frames
    j - 1 and j are out: samples [0, (length // H - 1) H).  At the end of the stream (final=True) the last frame,
    t = length // H, reflected at the end, and every sample up to `length` are out: 1 + length // H frames, as
    ops.n_frames(length)."""
    H = n_fft // 2
    if final:
        if length <= H:
            raise ValueError("a stream needs more than n_fft / 2 = %d samples (reflect padding), got %d" % (H, length))
        return 1 + length // H, length
    if length <= H:
        return 0, 0
    T = length // H
    return T, (T - 1) * H



def _check_params(n_fft, block, lambda_cor, lag):
    """The checks OnlineTangoStream and OnlineTangoPool share, before their own channel limit."""
    if n_fft not in N_FFTS:
        raise ValueError("n_fft must be 256, 512 or 1024")
    if not 1 <= int(block) <= 64:
        raise ValueError("block must be 1..64 frames")
    if not 0.0 <= float(lambda_cor) < 1.0:
        raise ValueError("lambda_cor must be in [0, 1)")
    if int(lag) == 0:
        raise NotImplementedError("lag = 0 filters a frame with its own block's statistics, whose masks arrive "
                                  "only after the block's later frames are out")
    if int(lag) < 0:
        raise ValueError("lag must be positive")


def _check_ref_mic(ref_mic, C):
    if not 0 <= int(ref_mic) < C:
        raise ValueError("ref_mic must be in 0..C-1")


def _cuda_device(device, what):
    """torch.device of the CUDA device `device` (None or no index: the current one); `what` names the caller."""
    device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    if device.type != "cuda":
        raise TypeError("the %s runs on a CUDA device, got %s" % (what, device))
    if device.index is None:
        device = torch.device("cuda", torch.cuda.current_device())
    return device


def _check_masks(masks, want, device):
    """(mask_z, mask_w) of a mask_fn result: float32 tensors of shape `want` on `device` (mask_w = None: mask_z)."""
    if not isinstance(masks, (tuple, list)) or len(masks) != 2:
        raise ValueError("mask_fn must return the pair (mask_z, mask_w)")
    mz, mw = masks
    mw = mz if mw is None else mw
    for m, name in ((mz, "mask_z"), (mw, "mask_w")):
        if not isinstance(m, torch.Tensor):
            raise ValueError("%s must be a tensor %s" % (name, want))
        if tuple(m.shape) != want:
            raise ValueError("%s shape %s, expected %s" % (name, tuple(m.shape), want))
        if m.dtype != torch.float32 or m.device != device:
            raise ValueError("%s must be float32 on %s" % (name, device))
    return mz, mw

class OnlineTangoStream:
    """B streams of K nodes x C microphones that start together and advance in lockstep; two-step recursive Tango
    (rank-`rank` GEVD filters), with the parameters of `online_tango`:

        s = OnlineTangoStream(B, K, C, n_fft=512, lambda_cor=0.95, block=8, lag=1)
        out = s.push(y_chunk, mask_fn)     # y_chunk [B, K, C, n] float32 CUDA, any n >= 0
        out = s.flush(mask_fn)             # end of the stream: the last frame and the remaining samples

    mask_fn(t0, Y, z_y, zn) -> (mask_z, mask_w) is called once for each run of newly completed frames [t0, t0 + f),
    after the run's step-1 outputs exist and before any later frame is filtered, with Y [B, K, C, f, F] (the STFT) and
    z_y, zn [B, K, f, F] (step 1).  It returns frame-major float32 masks [B, K, f, F]; mask_w = None means mask_z.
    Precomputed masks are a slice by t0; a causal estimator reads Y, z_y and zn.

    push and flush return dict(t0 = first frame of the call; z_y, zn, yf [B, K, f, F] of the frames the call
    completed; yf_time [B, K, s], the time samples of yf that became final), all fresh tensors.  A sample comes out
    n_fft / 2 to n_fft - 1 samples after it went in.  An exception raised inside push or flush (by mask_fn, or by a
    mask of the wrong shape) closes the stream."""

    def __init__(self, B, K, C, n_fft=512, lambda_cor=0.95, block=8, lag=1, mu=1.0, rank=1, ref_mic=0, R0=None,
                 device=None):
        B, K, C = int(B), int(K), int(C)
        if B < 1 or K < 1 or C < 1:
            raise ValueError("B, K and C must be positive")
        _check_params(n_fft, block, lambda_cor, lag)
        D = C + K - 1
        if D > 8:
            raise NotImplementedError("the stream covers C + K - 1 <= 8 channels, got %d (the whole-signal "
                                      "online_tango goes to 16)" % D)
        _check_ref_mic(ref_mic, C)
        if R0 is not None:
            if not isinstance(R0, (tuple, list)) or len(R0) != 2:
                raise ValueError("R0 must be the pair (R_ss, R_nn)")
            for r in R0:
                if not isinstance(r, torch.Tensor) or not r.is_cuda:
                    raise TypeError("R0 must hold CUDA tensors (disco_b200 has no CPU path)")
        device = _cuda_device(R0[0].device if device is None and R0 is not None else device, "stream")
        F, H, P = n_fft // 2 + 1, n_fft // 2, int(block)
        if R0 is not None:
            for r in R0:
                if r.dtype != torch.complex64 or tuple(r.shape) != (B, K, F, C, C) or r.device != device:
                    raise ValueError("R0 matrices must be complex64 [%d, %d, %d, %d, %d] on %s" % (B, K, F, C, C, device))
            R0 = tuple(r.contiguous().clone() for r in R0)
        self.B, self.K, self.C, self.D, self.F = B, K, C, D, F
        self.n_fft, self.block, self.lag = n_fft, P, int(lag)
        self.lambda_cor, self.mu, self.rank, self.ref_mic = float(lambda_cor), float(mu), rank, int(ref_mic)
        self.device = device
        f32, c64 = dict(dtype=torch.float32, device=device), dict(dtype=torch.complex64, device=device)
        self._hist = [torch.zeros((B, K, C, n_fft), **f32), torch.zeros((B, K, C, n_fft), **f32)]   # in, out
        self._none = torch.empty((B, K, C, 0), **f32)
        self._carry = torch.zeros((B, K, H), **f32)
        # the open block: its spectra, masks and (K > 1) step-1 outputs, written in place run by run
        self._Yblk = torch.zeros((B, K, C, P, F), **c64)
        self._m1 = torch.zeros((B, K, P, F), **f32)
        self._m2 = torch.zeros((B, K, P, F), **f32)
        self._zblk = torch.zeros((B, K, P, F), **c64) if K > 1 else None
        # carried statistics: step 1 from R0; step 2 from R0 for a single node, from zeros otherwise
        self._R1 = R0
        self._R2 = R0 if K == 1 else None
        # solved filters by block index, kept while a later block still uses them; pass-through stand-ins
        self._W1s, self._W2s = {}, {}
        self._pass1 = torch.zeros((B, K, 1, F, C), **c64)
        self._pass2 = torch.zeros((B, K, 1, F, D), **c64)
        self._L = self._T = self._S = 0
        self._closed = False

    # ---------------------------------------------------------------- state
    @property
    def W1(self):
        """Step-1 filters [B, K, F, C] of the last closed block (None before the first); block j's come into force for
        block j + lag."""
        return self._W1s[max(self._W1s)] if self._W1s else None

    @property
    def W2(self):
        """Step-2 filters [B, K, F, D] of the last closed block (None before the first)."""
        return self._W2s[max(self._W2s)] if self._W2s else None

    @property
    def samples_in(self):
        return self._L

    @property
    def frames_out(self):
        return self._T

    @property
    def samples_out(self):
        return self._S

    @property
    def closed(self):
        return self._closed

    # ---------------------------------------------------------------- public calls
    def push(self, y_chunk, mask_fn):
        """Append y_chunk [B, K, C, n] float32 (n >= 0) to every stream; returns what became final (class doc)."""
        self._check_open()
        if not isinstance(y_chunk, torch.Tensor) or not y_chunk.is_cuda:
            raise TypeError("y_chunk must be a CUDA tensor (disco_b200 has no CPU path)")
        if y_chunk.dtype != torch.float32:
            raise TypeError("y_chunk must be float32, got %s" % y_chunk.dtype)
        if y_chunk.dim() != 4 or tuple(y_chunk.shape[:3]) != (self.B, self.K, self.C):
            raise ValueError("y_chunk shape %s, expected (%d, %d, %d, n)" % (tuple(y_chunk.shape), self.B, self.K, self.C))
        if y_chunk.device != self.device:
            raise ValueError("y_chunk is on %s, the stream on %s" % (y_chunk.device, self.device))
        L1 = self._L + y_chunk.shape[-1]
        T1, S1 = emission(L1, self.n_fft)
        return self._run(y_chunk.contiguous(), L1, T1, S1, mask_fn, final=False)

    def flush(self, mask_fn):
        """End every stream: the last frame (reflected at the end), the final, partial block's statistics and filters,
        and the remaining time samples up to samples_in.  The stream is closed afterwards."""
        self._check_open()
        T1, S1 = emission(self._L, self.n_fft, final=True)   # ValueError for <= n_fft / 2 samples
        out = self._run(self._none, self._L, T1, S1, mask_fn, final=True)
        self._closed = True
        return out

    # ---------------------------------------------------------------- internals
    def _check_open(self):
        if self._closed:
            raise RuntimeError("the stream is closed (flushed, or an earlier push failed)")

    def _run(self, chunk, L1, T1, S1, mask_fn, final):
        try:
            return self._advance(chunk, L1, T1, S1, mask_fn, final)
        except BaseException:
            self._closed = True
            raise

    def _in_force(self, Ws, stand_in, j):
        """(W [B, K, 1, F, D], lag argument of filter_sum_blocks) for the frames of block j: the filter of block
        j - lag, or, while that does not exist, the kernel's own pass-through of the reference channel."""
        jw = j - self.lag
        return (stand_in, 1) if jw < 0 else (Ws[jw].unsqueeze(2), 0)

    def _close_block(self, j, nb):
        """Statistics and filters of block j once the masks of its nb frames are in (nb < block: the final, partial
        block, whose recursion step is lambda^nb, as in the whole-signal scan)."""
        P, lam, n_fft = self.block, self.lambda_cor, self.n_fft
        Yb, m1, m2, zb = self._Yblk, self._m1, self._m2, self._zblk
        if nb < P:
            Yb, m1, m2 = Yb[:, :, :, :nb].contiguous(), m1[:, :, :nb].contiguous(), m2[:, :, :nb].contiguous()
            zb = zb[:, :, :nb].contiguous() if zb is not None else None
        # scm_recursive writes fresh matrices, so its output never aliases the carried R0 it reads
        Rs1, Rn1 = ops.scm_recursive(Yb, m1, None, lam, P, 2, self._R1, n_fft)
        Rs2, Rn2 = ops.scm_recursive(Yb, m2, zb, lam, P, 2, self._R2, n_fft)
        self._R1, self._R2 = (Rs1[:, :, 0], Rn1[:, :, 0]), (Rs2[:, :, 0], Rn2[:, :, 0])
        self._W1s[j] = ops.mwf_solve(Rs1, Rn1, self.mu, "gevd", self.rank)[0][:, :, 0]
        self._W2s[j] = ops.mwf_solve(Rs2, Rn2, self.mu, "gevd", self.rank)[0][:, :, 0]
        for Ws in (self._W1s, self._W2s):
            for old in [i for i in Ws if i < j + 1 - self.lag]:
                del Ws[old]

    def _advance(self, chunk, L1, T1, S1, mask_fn, final):
        B, K, F, P, n_fft, ref = self.B, self.K, self.F, self.block, self.n_fft, self.ref_mic
        T0, S0 = self._T, self._S
        hist_in, hist_out = self._hist
        update = chunk.shape[-1] > 0          # the history moves with every sample that arrives
        yf_time = torch.empty((B, K, S1 - S0), dtype=torch.float32, device=self.device)
        parts = []
        if T1 == T0 and update:
            ops.stream_stft(hist_in, chunk, L1, T0, 0, n_fft, hist_out=hist_out)
        t = T0
        while t < T1:
            j, slot = divmod(t, P)
            f = min(T1, (j + 1) * P) - t
            last = t + f == T1
            Y = ops.stream_stft(hist_in, chunk, L1, t, f, n_fft, hist_out=hist_out if (last and update) else None,
                                Y_blk=self._Yblk, blk_slot=slot, final=final)
            W, lg = self._in_force(self._W1s, self._pass1, j)
            z, zn = ops.filter_sum_blocks(W, Y, None, P, lg, True, ref, n_fft)
            W, lg = self._in_force(self._W2s, self._pass2, j)
            yf, _ = ops.filter_sum_blocks(W, Y, z if K > 1 else None, P, lg, True, ref, n_fft)
            mz, mw = _check_masks(mask_fn(t, Y, z, zn), (B, K, f, F), self.device)
            self._m1[:, :, slot:slot + f].copy_(mz)
            self._m2[:, :, slot:slot + f].copy_(mw)
            if K > 1:
                self._zblk[:, :, slot:slot + f].copy_(z)
            if slot + f == P or (final and last):
                self._close_block(j, slot + f)
            ops.stream_istft(yf, self._carry, t, L1, n_fft, final=final and last, x=yf_time, x_first=S0)
            parts.append((z, zn, yf))
            t += f
        if update:
            self._hist.reverse()
        self._L, self._T, self._S = L1, T1, S1
        if not parts:
            empty = torch.empty((B, K, 0, F), dtype=torch.complex64, device=self.device)
            return {"t0": T0, "z_y": empty, "zn": empty.clone(), "yf": empty.clone(), "yf_time": yf_time}
        cat = (lambda i: parts[0][i]) if len(parts) == 1 else (lambda i: torch.cat([p[i] for p in parts], dim=2))
        return {"t0": T0, "z_y": cat(0), "zn": cat(1), "yf": cat(2), "yf_time": yf_time}


def pool_rounds(T0, T1, block):
    """The rounds of one call of OnlineTangoPool: slot s completes frames [T0[s], T1[s]); they are cut into runs that
    never cross a block boundary (multiples of `block`), and round r holds every slot's r-th run.  Returns int64 arrays
    (t0, n) of shape [R, S]: run r of slot s is frames [t0[r, s], t0[r, s] + n[r, s]); n[r, s] = 0 once slot s has no
    r-th run, and t0 is then where the slot stands (T1[s])."""
    T0, T1, P = np.asarray(T0, dtype=np.int64), np.asarray(T1, dtype=np.int64), int(block)
    if T0.shape != T1.shape or T0.ndim != 1 or P < 1 or np.any(T1 < T0) or np.any(T0 < 0):
        raise ValueError("need 0 <= T0 <= T1, one entry per slot, and block >= 1")
    b0 = (T0 // P + 1) * P                                   # the first block boundary after T0
    runs = np.where(T1 > T0, 1 + np.maximum(T1 - b0 + P - 1, 0) // P, 0)
    R = int(runs.max()) if runs.size else 0
    r = np.arange(R, dtype=np.int64)[:, None]
    start = np.where(r == 0, T0, b0 + (r - 1) * P)
    n = np.maximum(np.minimum(T1, b0 + r * P) - start, 0)
    return np.minimum(start, T1), n


class OnlineTangoPool:
    """S slots, each an independent online Tango stream of K nodes x C microphones that opens, advances and closes on
    its own; the parameters are those of OnlineTangoStream, and one pool has one geometry (D = C + K - 1 <= 16):

        pool = OnlineTangoPool(S, K, C, n_fft=512, lambda_cor=0.95, block=8, lag=1)
        pool.open(slots, R0=None)        # R0 = (R_ss, R_nn) complex64 [len(slots), K, F, C, C], or None
        out = pool.push(y, n, mask_fn)   # y [S, K, C, n_max] float32 CUDA; slot s gets y[s, ..., :n[s]]
        out = pool.close(slots, mask_fn) # the last frame (reflected at the end), the partial block, the last samples
        pool.filters(slot)               # (W1 [K, F, C], W2 [K, F, D]) of the slot's last closed block, or None

    For every slot, its outputs concatenated over the calls from open to close equal, value for value, those of
    OnlineTangoStream(1, K, C) fed the same samples (hence online_tango on the slot's whole signal and ops.istft of its
    yf), with the masks mask_fn returned -- whatever the other slots do, the slot's index, and the cut of its samples
    into pushes.  A slot's K C signals are paired into transforms inside the slot, as the single stream pairs them.

    mask_fn(t0, n_fr, Y, z_y, zn) -> (mask_z, mask_w) is called once per round: every slot's frames of the call are
    cut into runs that never cross its block boundary (pool_rounds), and round r holds every slot's r-th run.  t0 and
    n_fr are host int arrays [S] (n_fr[s] = 0: no frames of slot s in the round); Y is [S, K, C, f_max, F], z_y and zn
    [S, K, f_max, F]; the masks are float32 [S, K, f_max, F] (mask_w = None means mask_z).  Rows at or past n_fr[s] of
    Y are not defined, those of z_y and zn are 0, and those of the masks are never read.

    push and close return dict(t0, frames, s0, samples: host int arrays [S]; z_y, zn, yf [S, K, f_max, F]: the frames
    [t0[s], t0[s] + frames[s]) of slot s, exactly 0 from frames[s] on; yf_time [S, K, s_max]: its samples [s0[s],
    s0[s] + samples[s]) that became final, exactly 0 after them).  Invalid calls raise ValueError before any work and
    leave the pool as it was; an exception raised after work has started (by mask_fn, or a mask of the wrong shape)
    closes the slots the call advanced, and the others stay open and exact."""

    def __init__(self, S, K, C, n_fft=512, lambda_cor=0.95, block=8, lag=1, mu=1.0, rank=1, ref_mic=0, device=None):
        S, K, C = int(S), int(K), int(C)
        if S < 1 or K < 1 or C < 1:
            raise ValueError("S, K and C must be positive")
        _check_params(n_fft, block, lambda_cor, lag)
        D = C + K - 1
        if D > 16:
            raise NotImplementedError("the pool covers C + K - 1 <= 16 channels, got %d" % D)
        _check_ref_mic(ref_mic, C)
        if S > 65535:
            raise ValueError("at most 65535 slots")
        device = _cuda_device(device, "pool")
        self.S, self.K, self.C, self.D, self.F = S, K, C, D, n_fft // 2 + 1
        self.n_fft, self.block, self.lag = n_fft, int(block), int(lag)
        self.lambda_cor, self.mu, self.rank, self.ref_mic = float(lambda_cor), float(mu), rank, int(ref_mic)
        self.device = device
        # host state per slot
        self._open = np.zeros(S, dtype=bool)
        self._L = np.zeros(S, dtype=np.int64)          # samples in
        self._T = np.zeros(S, dtype=np.int64)          # frames out
        self._S = np.zeros(S, dtype=np.int64)          # time samples out
        self._par = np.zeros(S, dtype=np.int64)        # which history buffer holds the slot's last n_fft samples
        self._nclosed = np.zeros(S, dtype=np.int64)    # closed blocks
        self._bufs = False

    def _alloc(self):
        """Device state, allocated on the first open."""
        if self._bufs:
            return
        S, K, C, D, F, P, N, dev = self.S, self.K, self.C, self.D, self.F, self.block, self.n_fft, self.device
        f32, c64 = dict(dtype=torch.float32, device=dev), dict(dtype=torch.complex64, device=dev)
        self._hist = torch.zeros((2, S, K, C, N), **f32)
        self._carry = torch.zeros((S, K, N // 2), **f32)
        # the open block of every slot: its spectra, masks and (K > 1) step-1 outputs
        self._Yblk = torch.zeros((S, K, C, P, F), **c64)
        self._m1 = torch.zeros((S, K, P, F), **f32)
        self._m2 = torch.zeros((S, K, P, F), **f32)
        self._zblk = torch.zeros((S, K, P, F), **c64) if K > 1 else None
        # carried statistics (zeros stand for "none yet": the scan's R_(-1) is 0 either way)
        self._R1 = (torch.zeros((S, K, F, C, C), **c64), torch.zeros((S, K, F, C, C), **c64))
        self._R2 = (torch.zeros((S, K, F, D, D), **c64), torch.zeros((S, K, F, D, D), **c64))
        # ring of the last lag + 1 filters: block j's at j % (lag + 1).  Entries of blocks before the first hold the
        # pass-through of the reference channel, stored as (e_ref, -0) so that the kernel's conjugate is exactly the
        # weight vector of filter_sum_blocks' own pass-through.
        self._W1 = torch.zeros((S, self.lag + 1, K, F, C), **c64)
        self._W2 = torch.zeros((S, self.lag + 1, K, F, D), **c64)
        self._pass = []
        for d in (C, D):
            re = torch.zeros((K, F, d), **f32)
            re[..., self.ref_mic] = 1.0
            self._pass.append(torch.complex(re, torch.full_like(re, -0.0)))
        self._bufs = True

    # ---------------------------------------------------------------- state
    def is_open(self, slot):
        return bool(self._open[self._slot_list([slot])[0]])

    @property
    def samples_in(self):
        return self._L.copy()

    @property
    def frames_out(self):
        return self._T.copy()

    @property
    def samples_out(self):
        return self._S.copy()

    def filters(self, slot):
        """(W1 [K, F, C], W2 [K, F, D]) of the slot's last closed block (in force from block j + lag), or None before
        its first; kept after close until the slot is opened again."""
        s = int(self._slot_list([slot])[0])
        if self._nclosed[s] == 0:
            return None
        pos = int((self._nclosed[s] - 1) % (self.lag + 1))
        return self._W1[s, pos].clone(), self._W2[s, pos].clone()

    # ---------------------------------------------------------------- public calls
    def open(self, slots, R0=None):
        """Open free slots: every slot starts a new stream (history, block buffers, filters and iSTFT carry reset; the
        carried matrices from R0, or zeros).  R0 = (R_ss, R_nn), complex64 [len(slots), K, F, C, C]."""
        idx = self._slot_list(slots)
        if self._open[idx].any():
            raise ValueError("slot %d is already open" % int(idx[self._open[idx]][0]))
        K, C, F = self.K, self.C, self.F
        if R0 is not None:
            if not isinstance(R0, (tuple, list)) or len(R0) != 2:
                raise ValueError("R0 must be the pair (R_ss, R_nn)")
            for r in R0:
                if not isinstance(r, torch.Tensor) or not r.is_cuda:
                    raise TypeError("R0 must hold CUDA tensors (disco_b200 has no CPU path)")
                if r.dtype != torch.complex64 or tuple(r.shape) != (len(idx), K, F, C, C) or r.device != self.device:
                    raise ValueError("R0 matrices must be complex64 [%d, %d, %d, %d, %d] on %s"
                                     % (len(idx), K, F, C, C, self.device))
        if len(idx) == 0:
            return
        self._alloc()
        i = torch.from_numpy(idx).to(self.device)
        self._hist[:, i] = 0
        self._carry[i] = 0
        for buf in (self._Yblk, self._m1, self._m2, self._zblk):
            if buf is not None:
                buf[i] = 0
        for w in range(2):
            self._R1[w][i] = 0 if R0 is None else R0[w]
            self._R2[w][i] = R0[w] if (R0 is not None and K == 1) else 0   # step 2 of a single node starts from R0
        self._W1[i] = self._pass[0]
        self._W2[i] = self._pass[1]
        self._open[idx] = True
        for a in (self._L, self._T, self._S, self._par, self._nclosed):
            a[idx] = 0

    def push(self, y, n, mask_fn):
        """Append y[s, :, :, :n[s]] to slot s (y [S, K, C, n_max] float32 CUDA; n host ints, 0 <= n[s] <= n_max, and
        0 for free slots); returns what became final (class doc)."""
        if not isinstance(y, torch.Tensor):
            raise TypeError("y must be a CUDA tensor (disco_b200 has no CPU path)")
        if y.dim() != 4 or tuple(y.shape[:3]) != (self.S, self.K, self.C):
            raise ValueError("y shape %s, expected (%d, %d, %d, n_max)" % (tuple(y.shape), self.S, self.K, self.C))
        n_max = y.shape[-1]
        n = np.asarray(n)
        if n.dtype.kind not in "iu" or n.shape != (self.S,):
            raise ValueError("n must hold one integer per slot")
        n = n.astype(np.int64)
        if np.any(n < 0) or np.any(n > n_max):
            raise ValueError("every n[s] must lie in [0, %d]" % n_max)
        if np.any(n[~self._open] > 0):
            raise ValueError("samples pushed to free slot %d" % int(np.nonzero((n > 0) & ~self._open)[0][0]))
        if not y.is_cuda:
            raise TypeError("y must be a CUDA tensor (disco_b200 has no CPU path)")
        if y.dtype != torch.float32:
            raise TypeError("y must be float32, got %s" % y.dtype)
        if y.device != self.device:
            raise ValueError("y is on %s, the pool on %s" % (y.device, self.device))
        H = self.n_fft // 2
        L1 = self._L + n
        T1 = np.where(self._open & (L1 > H), L1 // H, self._T)
        S1 = np.where(self._open & (L1 > H), (L1 // H - 1) * H, self._S)
        return self._run(y.contiguous(), n, L1, T1, S1, np.zeros(self.S, dtype=bool), mask_fn)

    def close(self, slots, mask_fn):
        """End the streams of `slots`: the last frame (reflected at the end), the final, partial block's statistics
        and filters, and the remaining time samples up to samples_in.  The slots are free afterwards."""
        idx = self._slot_list(slots)
        if not self._open[idx].all():
            raise ValueError("slot %d is not open" % int(idx[~self._open[idx]][0]))
        H = self.n_fft // 2
        if np.any(self._L[idx] <= H):
            raise ValueError("a stream needs more than n_fft / 2 = %d samples (reflect padding)" % H)
        final = np.zeros(self.S, dtype=bool)
        final[idx] = True
        T1, S1 = self._T.copy(), self._S.copy()
        T1[idx] = 1 + self._L[idx] // H
        S1[idx] = self._L[idx]
        chunk = torch.empty((self.S, self.K, self.C, 0), dtype=torch.float32, device=self.device)
        out = self._run(chunk, np.zeros(self.S, dtype=np.int64), self._L.copy(), T1, S1, final, mask_fn)
        self._open[idx] = False
        return out

    # ---------------------------------------------------------------- internals
    def _slot_list(self, slots):
        idx = np.asarray(slots).reshape(-1)
        if idx.size and idx.dtype.kind not in "iu":
            raise ValueError("slots must be integers")
        idx = idx.astype(np.int64)
        if np.any(idx < 0) or np.any(idx >= self.S):
            raise ValueError("slots must lie in 0..%d" % (self.S - 1))
        if len(np.unique(idx)) != len(idx):
            raise ValueError("a slot is listed twice")
        return idx

    def _run(self, chunk, n, L1, T1, S1, final, mask_fn):
        touched = (n > 0) | (T1 > self._T) | final
        try:
            return self._advance(chunk, n, L1, T1, S1, final, mask_fn)
        except BaseException:
            self._open[touched] = False
            raise

    def _close_blocks(self, cl, nb, ci):
        """Statistics and filters of the open block of the slots `cl` (ci: the same indices on the device) once the
        masks of its nb[s] frames are in (nb < block: the final, partial block, whose recursion step is lambda^nb)."""
        P, lam, n_fft = self.block, self.lambda_cor, self.n_fft
        Yb, m1, m2 = self._Yblk[ci], self._m1[ci], self._m2[ci]
        zb = self._zblk[ci] if self.K > 1 else None
        R1 = (self._R1[0][ci], self._R1[1][ci])
        R2 = (self._R2[0][ci], self._R2[1][ci])
        Rs1, Rn1 = ops.scm_recursive(Yb, m1, None, lam, P, 2, R1, n_fft, frames=nb)
        Rs2, Rn2 = ops.scm_recursive(Yb, m2, zb, lam, P, 2, R2, n_fft, frames=nb)
        W1 = ops.mwf_solve(Rs1, Rn1, self.mu, "gevd", self.rank)[0][:, :, 0]
        W2 = ops.mwf_solve(Rs2, Rn2, self.mu, "gevd", self.rank)[0][:, :, 0]
        for R, new in ((self._R1, (Rs1, Rn1)), (self._R2, (Rs2, Rn2))):
            R[0][ci] = new[0][:, :, 0]
            R[1][ci] = new[1][:, :, 0]
        pos = torch.from_numpy(self._nclosed[cl] % (self.lag + 1)).to(self.device)
        self._W1[ci, pos] = W1
        self._W2[ci, pos] = W2
        self._nclosed[cl] += 1

    def _advance(self, chunk, n, L1, T1, S1, final, mask_fn):
        S, K, F, P, lag, n_fft, ref, dev = (self.S, self.K, self.F, self.block, self.lag, self.n_fft, self.ref_mic,
                                            self.device)
        T0, S0 = self._T.copy(), self._S.copy()
        frames, samples = T1 - T0, S1 - S0
        starts, runs = pool_rounds(T0, T1, P)
        c64 = dict(dtype=torch.complex64, device=dev)
        f_call = int(frames.max())
        out = [torch.zeros((S, K, f_call, F), **c64) for _ in range(3)]        # z_y, zn, yf
        yf_time = torch.zeros((S, K, int(samples.max())), dtype=torch.float32, device=dev)
        write = n > 0
        stft_rec = np.zeros((S, len(ops.STFT_SLOT_FIELDS)), dtype=np.int64)
        stft_rec[:, 0], stft_rec[:, 1], stft_rec[:, 5], stft_rec[:, 6] = L1, n, final, self._par
        istft_rec = np.zeros((S, len(ops.ISTFT_SLOT_FIELDS)), dtype=np.int64)
        istft_rec[:, 2], istft_rec[:, 4] = L1, S0
        if len(runs) == 0 and write.any():       # no frame completes: only the history moves
            stft_rec[:, 2], stft_rec[:, 7] = T0, write
            ops.stream_stft_slots(self._hist, chunk, stft_rec, 0, n_fft)
        for r in range(len(runs)):
            t0, nr = starts[r], runs[r]
            act = np.nonzero(nr)[0]
            fr, f = nr[act], int(nr.max())
            blk = np.where(nr > 0, t0 % P, 0)
            stft_rec[:, 2], stft_rec[:, 3], stft_rec[:, 4], stft_rec[:, 7] = t0, nr, blk, write if r == 0 else 0
            Y = ops.stream_stft_slots(self._hist, chunk, stft_rec, f, n_fft, Y_blk=self._Yblk)
            # one host -> device copy per round: active slots, ring positions, and the (slot, frame) pairs of the run
            s_idx = np.repeat(act, fr)
            a_idx = np.repeat(np.arange(len(act)), fr)
            i_idx = np.arange(len(s_idx)) - np.repeat(np.cumsum(fr) - fr, fr)
            pos = (t0[act] // P - lag) % (lag + 1)
            host = np.concatenate([act, pos, s_idx, a_idx, i_idx, blk[s_idx] + i_idx, (t0 - T0)[s_idx] + i_idx])
            d = torch.from_numpy(host).to(dev)
            na, nf = len(act), len(s_idx)
            ai, pi = d[:na], d[na:2 * na]
            si, aj, ii, bi, oi = (d[2 * na + k * nf:2 * na + (k + 1) * nf] for k in range(5))
            every = na == S
            Ya = Y if every else Y[ai]
            # step 1 and step 2 with the filter in force, W_(j - lag) (the pass-through stand-in before the first)
            z, zn = ops.filter_sum_blocks(self._W1[ai, pi].unsqueeze(2), Ya, None, P, 0, True, ref, n_fft, frames=fr)
            yf, _ = ops.filter_sum_blocks(self._W2[ai, pi].unsqueeze(2), Ya, z if K > 1 else None, P, 0, True, ref,
                                          n_fft, frames=fr)
            if every:
                zf, znf, yff = z, zn, yf
            else:
                zf, znf, yff = (torch.zeros((S, K, f, F), **c64) for _ in range(3))
                zf[ai], znf[ai], yff[ai] = z, zn, yf
            mz, mw = _check_masks(mask_fn(t0.copy(), nr.copy(), Y, zf, znf), (S, K, f, F), dev)
            self._m1[si, :, bi] = mz[si, :, ii]
            self._m2[si, :, bi] = mw[si, :, ii]
            if K > 1:
                self._zblk[si, :, bi] = z[aj, :, ii]
            for o, v in zip(out, (z, zn, yf)):
                o[si, :, oi] = v[aj, :, ii]
            ends = t0 + nr
            closing = (nr > 0) & ((blk + nr == P) | (final & (ends == T1)))
            if closing.any():
                cl = np.nonzero(closing)[0]
                self._close_blocks(cl, (blk + nr)[cl], ai if every and len(cl) == S else torch.from_numpy(cl).to(dev))
            istft_rec[:, 0], istft_rec[:, 1], istft_rec[:, 3] = t0, nr, final & (nr > 0) & (ends == T1)
            ops.stream_istft_slots(yff, self._carry, istft_rec, yf_time, n_fft)
        self._par = np.where(write, 1 - self._par, self._par)
        self._L, self._T, self._S = L1.copy(), T1.copy(), S1.copy()
        return {"t0": T0, "frames": frames, "s0": S0, "samples": samples, "z_y": out[0], "zn": out[1], "yf": out[2],
                "yf_time": yf_time}
