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
    stream_istft         the hop blocks of yf that became final (csrc/stream.cu)
"""
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
        D = C + K - 1
        if D > 8:
            raise NotImplementedError("the stream covers C + K - 1 <= 8 channels, got %d (the whole-signal "
                                      "online_tango goes to 16)" % D)
        if not 0 <= int(ref_mic) < C:
            raise ValueError("ref_mic must be in 0..C-1")
        if R0 is not None:
            if not isinstance(R0, (tuple, list)) or len(R0) != 2:
                raise ValueError("R0 must be the pair (R_ss, R_nn)")
            for r in R0:
                if not isinstance(r, torch.Tensor) or not r.is_cuda:
                    raise TypeError("R0 must hold CUDA tensors (disco_b200 has no CPU path)")
        if device is None:
            device = R0[0].device if R0 is not None else torch.device("cuda", torch.cuda.current_device())
        device = torch.device(device)
        if device.type != "cuda":
            raise TypeError("the stream runs on a CUDA device, got %s" % device)
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
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

    def _masks(self, masks, f):
        if not isinstance(masks, (tuple, list)) or len(masks) != 2:
            raise ValueError("mask_fn must return the pair (mask_z, mask_w)")
        mz, mw = masks
        mw = mz if mw is None else mw
        want = (self.B, self.K, f, self.F)
        for m, name in ((mz, "mask_z"), (mw, "mask_w")):
            if not isinstance(m, torch.Tensor):
                raise ValueError("%s must be a tensor %s" % (name, want))
            if tuple(m.shape) != want:
                raise ValueError("%s shape %s, expected %s" % (name, tuple(m.shape), want))
            if m.dtype != torch.float32 or m.device != self.device:
                raise ValueError("%s must be float32 on %s" % (name, self.device))
        return mz, mw

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
            mz, mw = self._masks(mask_fn(t, Y, z, zn), f)
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
