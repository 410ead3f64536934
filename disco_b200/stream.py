"""Online Tango as a stream: push audio chunk by chunk, get the beamformed samples back about a frame later.

`online_tango` (online.py) runs the causal variant of Tango over a finished recording.  `OnlineTangoStream` runs the
same computation on audio as it arrives, and a causal mask estimator may compute the masks of each run of frames from
the frames just analysed (the step's own STFT and step-1 outputs).  Whatever the chunk sizes, the outputs equal
`online_tango` on the whole signal (with the masks the estimator returned, and the same options) and `ops.istft` of its
`yf`, value for value: every stage is a deterministic kernel that works per frame or per block of frames, so the stream
evaluates the same operations in the same order, only at different times.  Channel stacks D = C + K - 1 up to 16 run,
as in `online_tango` (9..16 with wide=True); at D >= 9 the block's statistics come from the staged scan, which splits
exactly at a block.

Per push, for every run of newly completed frames (a run never crosses a block boundary):
    stream_stft          the run's frames from the carried last n_fft samples and the chunk (csrc/stream.cu); with
                         clean components, those of s and n as well
    filter_sum_blocks    step 1 (z, zn) and step 2 (yf) with the filters in force, W_(j - lag) for block j; with clean
                         components also z_s, z_n, sf, nf
    mask_fn / tf_mask    the run's masks (from the estimator, or the oracle masks of the clean components), kept in the
                         open block's buffers
    scm_recursive        once a block's last masks are in: its statistics from the carried matrices (apply_mask and
                         tf_mask first for the exchange modes other than 'local'),
    mwf_solve            and the block's filters W1_j, W2_j
    stream_istft         the hop blocks of yf (with clean components: of the six time signals) that became final
"""
import numpy as np
import torch

from . import ops
from .tango import _ORACLE_SIGS, _clean_masks, _mask_kind, _ref_plane, _z_for_stats

N_FFTS = (256, 512, 1024)
# the time signals of a stream with clean components, in post.to_time's order (their iSTFT pairs signals across them)
TIME_NAMES = ("yf", "z_y", "sf", "nf", "z_s", "z_n")


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


def _check_options(filter_type, rank, mask_for_z, clean, vads):
    """online_tango's argument errors (tango._check_sources, the solver's filter check) for a stream, and the mask
    sources a stream cannot take, raised before any device work."""
    if mask_for_z is None:
        raise TypeError("argument of type 'NoneType' is not iterable")   # as tango._check_sources
    if not isinstance(mask_for_z, str):
        raise TypeError("mask_for_z must be a string, got %r" % (mask_for_z,))
    if mask_for_z == "use_oracle_sigs":
        raise NotImplementedError(_ORACLE_SIGS)
    if not clean and mask_for_z in ("compressed", "use_oracle_refs", "use_oracle_zs"):
        raise ValueError("mask_for_z=%r needs the clean components s and n" % mask_for_z)
    ops._filter_args(filter_type, rank)                 # AttributeError for an unknown filter, as the solver
    if vads is None:
        return
    if not isinstance(vads, (tuple, list)) or len(vads) != 2:
        raise ValueError("vads must be the pair (step-1 mask type, step-2 mask type)")
    for v in vads:
        kind = _mask_kind(v)                            # ValueError for an unknown type
        if kind == "ivad":
            raise ValueError("'ivad' masks take a quantile over the whole signal and cannot stream")
        if kind == "dnn":
            raise ValueError("network masks ('crnn' / 'rnn') come in through mask_fn")


def _split_scans(Xs, Xn, Zs, Zn, mask, lambda_cor, block, R0, n_fft, frames=None):
    """The statistics of online._online_mwf_split on a run of blocks: R_ss the unweighted recursive scan of [Xs ; Zs],
    R_nn that of [Xn ; Zn] (Xs, Xn first scaled by mask and 1 - mask when a mask is given), seeded by R0 = (R_ss,
    R_nn) of the block before, or None.  Returns (R_ss, R_nn) [B, K, J, F, D, D]."""
    if mask is not None:
        Xs, Xn = ops.apply_mask(Xs, mask, False), ops.apply_mask(Xn, mask, True)
    r0s, r0n = (None, None) if R0 is None else ((R0[0], R0[0]), (R0[1], R0[1]))   # the second matrix is not used
    Rss, _ = ops.scm_recursive(Xs, None, Zs, lambda_cor, block, 2, r0s, n_fft, frames=frames)
    Rnn, _ = ops.scm_recursive(Xn, None, Zn, lambda_cor, block, 2, r0n, n_fft, frames=frames)
    return Rss, Rnn


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
    """B streams of K nodes x C microphones (D = C + K - 1 <= 8, or <= 16 with wide=True) that start together and
    advance in lockstep; two-step recursive Tango with the parameters and options of `online_tango`:

        s = OnlineTangoStream(B, K, C, n_fft=512, lambda_cor=0.95, block=8, lag=1)
        out = s.push(y_chunk, mask_fn)     # y_chunk [B, K, C, n] float32 CUDA, any n >= 0
        out = s.flush(mask_fn)             # end of the stream: the last frame and the remaining samples

    mask_fn(t0, Y, z_y, zn) -> (mask_z, mask_w) is called once for each run of newly completed frames [t0, t0 + f),
    after the run's step-1 outputs exist and before any later frame is filtered, with Y [B, K, C, f, F] (the STFT) and
    z_y, zn [B, K, f, F] (step 1).  It returns frame-major float32 masks [B, K, f, F]; mask_w = None means mask_z.
    Precomputed masks are a slice by t0; a causal estimator reads Y, z_y and zn.  A call that completes no frame needs
    no mask_fn.

    filter_type, mu and rank reach both solves; mask_for_z is online_tango's exchange mode ('local', 'distant', and
    any other string but the ones below: 'previous', the unmasked z in both statistics).  With clean=True every push
    also takes the clean components of y, push(y_chunk, mask_fn, s_chunk=s, n_chunk=n) with s, n shaped like y_chunk,
    which allows 'compressed' (z masked by the vads[0] mask of z_s, z_n; 'irm1' without vads), 'use_oracle_refs' and
    'use_oracle_zs'.  vads = (step-1 type, step-2 type) of 'irmX' / 'ibmX' / 'iamX' builds the masks from the clean
    components as online_tango(masks=None) does (step 1 of microphone ref_mic, step 2 of microphone 0) and implies
    clean=True; push and flush then take no mask_fn.  Masks over the whole signal ('ivad') or from a network cannot be
    built by the stream; a network's masks come in through mask_fn.

    wide=True opts in to the channel stacks D = 9..16 (the MEETIT geometry of 8 nodes x 2 mics among them); without
    it a stack above 8 raises NotImplementedError, as the stream always has.  Their block statistics come from the
    staged scan, which reads only the upper triangle and the real diagonal of R0 (a given R0 of C >= 9 microphones, or
    the carried matrices, which are Hermitian with a real diagonal), where the D <= 8 scan reads every entry.

    push and flush return dict(t0 = first frame of the call; z_y, zn, yf [B, K, f, F] of the frames the call
    completed; yf_time [B, K, s], the time samples of yf that became final), all fresh tensors.  With clean components
    they also hold z_s, z_n, sf, nf [B, K, f, F] and the time samples <name>_time of every name of TIME_NAMES, equal to
    post.to_time(out, L, n_fft, layout="TF") of the whole-signal outputs (one iSTFT over the six signals, so yf_time
    equals ops.istft of yf alone when B K is even); with vads also masks_z, mask_w [B, K, f, F].  A sample comes out
    n_fft / 2 to n_fft - 1 samples after it went in.  An exception raised inside push or flush (by mask_fn, or by a
    mask of the wrong shape) closes the stream."""

    def __init__(self, B, K, C, n_fft=512, lambda_cor=0.95, block=8, lag=1, mu=1.0, rank=1, ref_mic=0, R0=None,
                 device=None, *, filter_type="gevd", mask_for_z="local", clean=False, vads=None, wide=False):
        B, K, C = int(B), int(K), int(C)
        if B < 1 or K < 1 or C < 1:
            raise ValueError("B, K and C must be positive")
        _check_params(n_fft, block, lambda_cor, lag)
        D = C + K - 1
        if D > 16:
            raise NotImplementedError("the stream covers C + K - 1 <= 16 channels, got %d" % D)
        if D > 8 and not wide:
            raise NotImplementedError("C + K - 1 = %d: the stream covers 9..16 channels with wide=True "
                                      "(<= 8 without)" % D)
        _check_ref_mic(ref_mic, C)
        clean = bool(clean) or vads is not None
        _check_options(filter_type, rank, mask_for_z, clean, vads)
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
        self.filter_type, self.mask_for_z, self.clean = filter_type, mask_for_z, clean
        self.vads = None if vads is None else tuple(vads)
        self.device = device
        f32, c64 = dict(dtype=torch.float32, device=device), dict(dtype=torch.complex64, device=device)
        pair = lambda: [torch.zeros((B, K, C, n_fft), **f32), torch.zeros((B, K, C, n_fft), **f32)]   # in, out
        self._hist = pair()
        self._hist_sn = (pair(), pair()) if clean else None
        self._none = torch.empty((B, K, C, 0), **f32)
        # one iSTFT carry per time signal: yf, or the six of TIME_NAMES
        self._carry = torch.zeros((len(TIME_NAMES), B, K, H) if clean else (B, K, H), **f32)
        # the open block: its spectra, masks and (K > 1) step-1 outputs, written in place run by run; the clean
        # spectra for the 'use_oracle_*' statistics, z_s and z_n for the exchange modes that read them
        self._oracle1 = "use_oracle_" in mask_for_z
        self._Yblk = torch.zeros((B, K, C, P, F), **c64)
        self._m1 = torch.zeros((B, K, P, F), **f32)
        self._m2 = torch.zeros((B, K, P, F), **f32)
        self._zblk = torch.zeros((B, K, P, F), **c64) if K > 1 else None
        self._SNblk = tuple(torch.zeros((B, K, C, P, F), **c64) for _ in range(2)) if self._oracle1 else None
        self._zsnblk = None
        if K > 1 and mask_for_z in ("compressed", "use_oracle_zs"):
            self._zsnblk = tuple(torch.zeros((B, K, P, F), **c64) for _ in range(2))
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
    def push(self, y_chunk, mask_fn=None, *, s_chunk=None, n_chunk=None):
        """Append y_chunk [B, K, C, n] float32 (n >= 0) to every stream, and s_chunk, n_chunk (its clean components,
        shaped like it) to a stream with clean components; returns what became final (class doc)."""
        self._check_open()
        self._check_chunk(y_chunk, "y_chunk")
        if self.clean:
            if s_chunk is None or n_chunk is None:
                raise ValueError("a stream with clean components takes s_chunk and n_chunk with every push")
            for x, name in ((s_chunk, "s_chunk"), (n_chunk, "n_chunk")):
                self._check_chunk(x, name)
                if x.shape != y_chunk.shape:
                    raise ValueError("%s shape %s, y_chunk %s" % (name, tuple(x.shape), tuple(y_chunk.shape)))
            sn = (s_chunk.contiguous(), n_chunk.contiguous())
        elif s_chunk is not None or n_chunk is not None:
            raise ValueError("s_chunk and n_chunk go to a stream made with clean=True")
        else:
            sn = None
        L1 = self._L + y_chunk.shape[-1]
        T1, S1 = emission(L1, self.n_fft)
        self._check_mask_fn(mask_fn, T1 > self._T)
        return self._run(y_chunk.contiguous(), sn, L1, T1, S1, mask_fn, final=False)

    def flush(self, mask_fn=None):
        """End every stream: the last frame (reflected at the end), the final, partial block's statistics and filters,
        and the remaining time samples up to samples_in.  The stream is closed afterwards."""
        self._check_open()
        T1, S1 = emission(self._L, self.n_fft, final=True)   # ValueError for <= n_fft / 2 samples
        self._check_mask_fn(mask_fn, True)
        sn = (self._none, self._none) if self.clean else None
        out = self._run(self._none, sn, self._L, T1, S1, mask_fn, final=True)
        self._closed = True
        return out

    # ---------------------------------------------------------------- internals
    def _check_open(self):
        if self._closed:
            raise RuntimeError("the stream is closed (flushed, or an earlier push failed)")

    def _check_chunk(self, x, name):
        if not isinstance(x, torch.Tensor) or not x.is_cuda:
            raise TypeError("%s must be a CUDA tensor (disco_b200 has no CPU path)" % name)
        if x.dtype != torch.float32:
            raise TypeError("%s must be float32, got %s" % (name, x.dtype))
        if x.dim() != 4 or tuple(x.shape[:3]) != (self.B, self.K, self.C):
            raise ValueError("%s shape %s, expected (%d, %d, %d, n)" % (name, tuple(x.shape), self.B, self.K, self.C))
        if x.device != self.device:
            raise ValueError("%s is on %s, the stream on %s" % (name, x.device, self.device))

    def _check_mask_fn(self, mask_fn, frames):
        """The mask source of a call that completes frames (`frames`): mask_fn, or vads, never both."""
        if self.vads is not None and mask_fn is not None:
            raise ValueError("the stream builds its masks from vads: no mask_fn")
        if self.vads is None and mask_fn is None and frames:
            raise ValueError("mask_fn is needed: the call completes frames")

    def _run(self, chunk, sn, L1, T1, S1, mask_fn, final):
        try:
            return self._advance(chunk, sn, L1, T1, S1, mask_fn, final)
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
        block, whose recursion step is lambda^nb, as in the whole-signal scan).  The statistics are online_tango's
        for the stream's mask_for_z: the masked scans for 'local', the split scans of [mask Y ; z_rs] and
        [(1 - mask) Y ; z_rn] otherwise, and those of S and N for step 1 under 'use_oracle_*'."""
        P, lam, n_fft, K = self.block, self.lambda_cor, self.n_fft, self.K
        cut = (lambda b: b) if nb == P else (lambda b: None if b is None else b[..., :nb, :].contiguous())
        Yb, m1, m2, zb = cut(self._Yblk), cut(self._m1), cut(self._m2), cut(self._zblk)
        Sb, Nb = (cut(b) for b in self._SNblk) if self._SNblk is not None else (None, None)
        zsb, znb = (cut(b) for b in self._zsnblk) if self._zsnblk is not None else (None, None)
        # scm_recursive writes fresh matrices, so its output never aliases the carried R0 it reads
        if self._oracle1:
            Rs1, Rn1 = _split_scans(Sb, Nb, None, None, None, lam, P, self._R1, n_fft)
        else:
            Rs1, Rn1 = ops.scm_recursive(Yb, m1, None, lam, P, 2, self._R1, n_fft)
        if self.mask_for_z == "local":
            Rs2, Rn2 = ops.scm_recursive(Yb, m2, zb, lam, P, 2, self._R2, n_fft)
        else:
            # what the other nodes contribute; a single node has none (online_tango reads its own channels only)
            z_rs = z_rn = None
            if K > 1:
                kind = self.vads[0] if self.vads is not None else "irm1"
                z_rs, z_rn = _z_for_stats(self.mask_for_z, (kind, kind), zb, m2, zsb, znb,
                                          lambda: (_ref_plane(Sb, self.ref_mic), _ref_plane(Nb, self.ref_mic)))
            Rs2, Rn2 = _split_scans(Yb, Yb, z_rs, z_rn, m2, lam, P, self._R2, n_fft)
        self._R1, self._R2 = (Rs1[:, :, 0], Rn1[:, :, 0]), (Rs2[:, :, 0], Rn2[:, :, 0])
        self._W1s[j] = ops.mwf_solve(Rs1, Rn1, self.mu, self.filter_type, self.rank)[0][:, :, 0]
        self._W2s[j] = ops.mwf_solve(Rs2, Rn2, self.mu, self.filter_type, self.rank)[0][:, :, 0]
        for Ws in (self._W1s, self._W2s):
            for old in [i for i in Ws if i < j + 1 - self.lag]:
                del Ws[old]

    def _advance(self, chunk, sn, L1, T1, S1, mask_fn, final):
        B, K, F, P, n_fft, ref = self.B, self.K, self.F, self.block, self.n_fft, self.ref_mic
        T0, S0 = self._T, self._S
        hist_in, hist_out = self._hist
        clean = sn is not None
        update = chunk.shape[-1] > 0          # the history moves with every sample that arrives
        x_time = torch.empty(((len(TIME_NAMES),) if clean else ()) + (B, K, S1 - S0), dtype=torch.float32,
                             device=self.device)
        names = ["z_y", "zn", "yf"] + (["z_s", "z_n", "sf", "nf"] if clean else []) + \
            (["masks_z", "mask_w"] if self.vads is not None else [])
        parts = []
        if T1 == T0 and update:
            ops.stream_stft(hist_in, chunk, L1, T0, 0, n_fft, hist_out=hist_out)
            if clean:
                for x, (h_in, h_out) in zip(sn, self._hist_sn):
                    ops.stream_stft(h_in, x, L1, T0, 0, n_fft, hist_out=h_out)
        t = T0
        while t < T1:
            j, slot = divmod(t, P)
            f = min(T1, (j + 1) * P) - t
            last = t + f == T1
            Y = ops.stream_stft(hist_in, chunk, L1, t, f, n_fft, hist_out=hist_out if (last and update) else None,
                                Y_blk=self._Yblk, blk_slot=slot, final=final)
            if clean:
                # S, N: one transform each, as online_tango takes them (the pairing of signals decides the bits)
                S, N = (ops.stream_stft(h_in, x, L1, t, f, n_fft, hist_out=h_out if (last and update) else None,
                                        Y_blk=None if self._SNblk is None else self._SNblk[i], blk_slot=slot,
                                        final=final)
                        for i, (x, (h_in, h_out)) in enumerate(zip(sn, self._hist_sn)))
            W1, lg1 = self._in_force(self._W1s, self._pass1, j)
            z, zn = ops.filter_sum_blocks(W1, Y, None, P, lg1, True, ref, n_fft)
            W2, lg2 = self._in_force(self._W2s, self._pass2, j)
            yf, _ = ops.filter_sum_blocks(W2, Y, z if K > 1 else None, P, lg2, True, ref, n_fft)
            if self.vads is None:
                mz, mw = _check_masks(mask_fn(t, Y, z, zn), (B, K, f, F), self.device)
            else:
                # tf_mask is elementwise, so the run's masks are those of the whole signal; S stands in for the time
                # signal, which only 'ivad' reads
                mz, mw = _clean_masks(S, N, S, self.vads, ref, n_fft)
            self._m1[:, :, slot:slot + f].copy_(mz)
            self._m2[:, :, slot:slot + f].copy_(mw)
            if K > 1:
                self._zblk[:, :, slot:slot + f].copy_(z)
            part = [z, zn, yf]
            if clean:
                # the diagnostics of online_tango: W1 on S, N; W2 on [S_own ; z_s], [N_own ; z_n]
                z_s = ops.filter_sum_blocks(W1, S, None, P, lg1, True, ref, n_fft)[0]
                z_n = ops.filter_sum_blocks(W1, N, None, P, lg1, True, ref, n_fft)[0]
                sf = ops.filter_sum_blocks(W2, S, z_s if K > 1 else None, P, lg2, True, ref, n_fft)[0]
                nf = ops.filter_sum_blocks(W2, N, z_n if K > 1 else None, P, lg2, True, ref, n_fft)[0]
                if self._zsnblk is not None:
                    self._zsnblk[0][:, :, slot:slot + f].copy_(z_s)
                    self._zsnblk[1][:, :, slot:slot + f].copy_(z_n)
                part += [z_s, z_n, sf, nf]
            if self.vads is not None:
                part += [mz, mw]
            if slot + f == P or (final and last):
                self._close_block(j, slot + f)
            if clean:
                sig = dict(zip(names, part))
                X = torch.stack([sig[nm] for nm in TIME_NAMES])          # post.to_time's stack: one pairing
                ops.stream_istft(X, self._carry, t, L1, n_fft, final=final and last, x=x_time, x_first=S0)
            else:
                ops.stream_istft(yf, self._carry, t, L1, n_fft, final=final and last, x=x_time, x_first=S0)
            parts.append(part)
            t += f
        if update:
            self._hist.reverse()
            if clean:
                for h in self._hist_sn:
                    h.reverse()
        self._L, self._T, self._S = L1, T1, S1
        out = {"t0": T0}
        for i, nm in enumerate(names):
            if not parts:
                dt = torch.float32 if nm in ("masks_z", "mask_w") else torch.complex64
                out[nm] = torch.empty((B, K, 0, F), dtype=dt, device=self.device)
            elif len(parts) == 1:
                out[nm] = parts[0][i]
            else:
                out[nm] = torch.cat([p[i] for p in parts], dim=2)
        if clean:
            for i, nm in enumerate(TIME_NAMES):
                out[nm + "_time"] = x_time[i]
        else:
            out["yf_time"] = x_time
        return out


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
    its own; the parameters are those of OnlineTangoStream, filter_type and the exchange modes that need no clean
    components ('local', 'distant', 'previous') included, and one pool has one geometry (D = C + K - 1 <= 16):

        pool = OnlineTangoPool(S, K, C, n_fft=512, lambda_cor=0.95, block=8, lag=1)
        pool.open(slots, R0=None)        # R0 = (R_ss, R_nn) complex64 [len(slots), K, F, C, C], or None
        out = pool.push(y, n, mask_fn)   # y [S, K, C, n_max] float32 CUDA; slot s gets y[s, ..., :n[s]]
        out = pool.close(slots, mask_fn) # the last frame (reflected at the end), the partial block, the last samples
        pool.filters(slot)               # (W1 [K, F, C], W2 [K, F, D]) of the slot's last closed block, or None

    For every slot, its outputs concatenated over the calls from open to close equal, value for value, those of
    OnlineTangoStream(1, K, C) with the same options fed the same samples (hence online_tango on the slot's whole
    signal and ops.istft of its yf), with the masks mask_fn returned -- whatever the other slots do, the slot's index,
    and the cut of its samples into pushes.  A slot's K C signals are paired into transforms inside the slot, as the single stream pairs them.

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

    def __init__(self, S, K, C, n_fft=512, lambda_cor=0.95, block=8, lag=1, mu=1.0, rank=1, ref_mic=0, device=None,
                 *, filter_type="gevd", mask_for_z="local"):
        S, K, C = int(S), int(K), int(C)
        if S < 1 or K < 1 or C < 1:
            raise ValueError("S, K and C must be positive")
        _check_params(n_fft, block, lambda_cor, lag)
        D = C + K - 1
        if D > 16:
            raise NotImplementedError("the pool covers C + K - 1 <= 16 channels, got %d" % D)
        _check_ref_mic(ref_mic, C)
        _check_options(filter_type, rank, mask_for_z, False, None)
        if S > 65535:
            raise ValueError("at most 65535 slots")
        device = _cuda_device(device, "pool")
        self.S, self.K, self.C, self.D, self.F = S, K, C, D, n_fft // 2 + 1
        self.n_fft, self.block, self.lag = n_fft, int(block), int(lag)
        self.lambda_cor, self.mu, self.rank, self.ref_mic = float(lambda_cor), float(mu), rank, int(ref_mic)
        self.filter_type, self.mask_for_z = filter_type, mask_for_z
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
        if self.mask_for_z == "local":
            Rs2, Rn2 = ops.scm_recursive(Yb, m2, zb, lam, P, 2, R2, n_fft, frames=nb)
        else:
            z_rs, z_rn = (None, None) if zb is None else _z_for_stats(self.mask_for_z, None, zb, m2, None, None, None)
            Rs2, Rn2 = _split_scans(Yb, Yb, z_rs, z_rn, m2, lam, P, R2, n_fft, frames=nb)
        W1 = ops.mwf_solve(Rs1, Rn1, self.mu, self.filter_type, self.rank)[0][:, :, 0]
        W2 = ops.mwf_solve(Rs2, Rn2, self.mu, self.filter_type, self.rank)[0][:, :, 0]
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
