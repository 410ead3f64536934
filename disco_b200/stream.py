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

Ragged arrays.  C may also be a sequence of K per-node microphone counts (`channels`); the inputs are then packed as
ragged.py packs them, [B, M, n] with M = sum(channels) and node k on rows off_k .. off_k + C_k - 1.  The nodes of
one count form a group, and every per-node stage above runs once per group on [B, n_C, C, ...]: the STFT of each
group from its own history (so signals pair inside the group, as online_tango_ragged's per-group transforms pair
them), step 1, step 2 with the z of all K nodes and the group's node_sel, and the block statistics and solves.  The
buffers that span all K nodes (masks, z, outputs) are assembled with index_copy.  An int C is the one-group case.
"""
import numpy as np
import torch

from . import ops, stream_state
from .ragged import _Layout, _group_R0
from .tango import _ORACLE_SIGS, _mask_kind, _ref_plane, _step1_mask, _step2_mask, _z_for_stats

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


def _split_scans(Xs, Xn, Zs, Zn, mask, lambda_cor, block, R0, n_fft, frames=None, node_sel=None):
    """The statistics of online._online_mwf_split on a run of blocks: R_ss the unweighted recursive scan of [Xs ; Zs],
    R_nn that of [Xn ; Zn] (Xs, Xn first scaled by mask and 1 - mask when a mask is given), seeded by R0 = (R_ss,
    R_nn) of the block before, or None; node_sel: the nodes Xs holds when Zs spans more.  Returns (R_ss, R_nn)
    [B, K, J, F, D, D]."""
    if mask is not None:
        Xs, Xn = ops.apply_mask(Xs, mask, False), ops.apply_mask(Xn, mask, True)
    r0s, r0n = (None, None) if R0 is None else ((R0[0], R0[0]), (R0[1], R0[1]))   # the second matrix is not used
    Rss, _ = ops.scm_recursive(Xs, None, Zs, lambda_cor, block, 2, r0s, n_fft, node_sel=node_sel, frames=frames)
    Rnn, _ = ops.scm_recursive(Xn, None, Zn, lambda_cor, block, 2, r0n, n_fft, node_sel=node_sel, frames=frames)
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


def _is_ragged(C):
    """C given as per-node microphone counts (a sequence) rather than one count for every node."""
    if isinstance(C, (str, bytes)):
        return False
    if isinstance(C, (torch.Tensor, np.ndarray)):
        return C.ndim > 0
    return hasattr(C, "__len__")


class _Group:
    """The nodes of one microphone count C (all K nodes when C is an int), and the state a stream or pool keeps for
    them.  sel is the node_sel of its step-2 launches: None when the group holds every node.  Its device indices
    are built on first use (a pool touches the device on its first open only)."""

    def __init__(self, C, nodes, K, lay, device):
        self.C, self.nodes, self.n, self.D = C, list(nodes), len(nodes), C + K - 1
        self.sel = None if self.n == K else self.nodes
        self._lay, self._device = lay, device

    @property
    def idx(self):
        """The group's nodes as a device index."""
        return self._lay.node_index(self.C, self._device)

    @property
    def rows(self):
        """The group's packed rows as a device index, node-major."""
        return self._lay.rows(self.C, self._device)


class _Geometry:
    """The channel layout of a stream or a pool: C an int (K nodes x C microphones, inputs [B, K, C, n]) or a sequence
    of K counts (channels: the packed inputs [B, M, n] of ragged.py).  Either way the nodes of one count form a
    group, and the per-node stages run once per group; these helpers move tensors between the groups and the
    layouts that span all K nodes."""

    def _set_geometry(self, K, C, ref_mic, what, wide):
        """Checks C (and ref_mic, and D against `wide`) before any device work; sets channels (None for an int C),
        C, M, D and the layout.  Errors: the stream's own for an int C, ragged._Layout's for a sequence."""
        ragged = _is_ragged(C)
        if ragged:
            lay = _Layout(C, None, ref_mic)            # counts, K <= 16, D <= 16, ref_mic on every node
            if lay.K != K:
                raise ValueError("channels holds %d counts for K = %d nodes" % (lay.K, K))
            self.channels, self.C = list(lay.channels), tuple(lay.channels)
            D = max(lay.channels) + K - 1
        else:
            C = int(C)
            D = C + K - 1
            if D > 16:
                raise NotImplementedError("the %s covers C + K - 1 <= 16 channels, got %d" % (what, D))
        if D > 8 and not wide:
            raise NotImplementedError("C + K - 1 = %d: the stream covers 9..16 channels with wide=True "
                                      "(<= 8 without)" % D)
        if not ragged:
            _check_ref_mic(ref_mic, C)
            lay = _Layout([C] * K, None, int(ref_mic))
            self.channels, self.C = None, C
        self.K, self.D, self.M, self._lay = K, D, sum(lay.channels), lay

    def _make_groups(self, device):
        self._groups = [_Group(C, nodes, self.K, self._lay, device) for C, nodes in self._lay.groups]

    @property
    def nodes(self):
        """{C: the node indices of count C}, as online_tango_ragged returns them."""
        return {g.C: list(g.nodes) for g in self._groups}

    def _lead(self, first):
        """The leading shape of an input: (first, K, C), or (first, M) packed."""
        return (first, self.K, self.C) if self.channels is None else (first, self.M)

    def _split(self, x):
        """An input [B, K, C, ...] or packed [B, M, ...] (contiguous) -> per group [B, n_C, C, ...]."""
        if self.channels is None:
            return [x]
        return [(x if g.n == self.K else x.index_select(1, g.rows)).view(x.shape[0], g.n, g.C, *x.shape[2:])
                for g in self._groups]

    def _join(self, parts):
        """Per group [B, n_C, ...] -> [B, K, ...] over all nodes (one index_copy per group)."""
        if len(parts) == 1:
            return parts[0]
        p0 = parts[0]
        out = torch.empty((p0.shape[0], self.K) + tuple(p0.shape[2:]), dtype=p0.dtype, device=p0.device)
        for g, p in zip(self._groups, parts):
            out.index_copy_(1, g.idx, p)
        return out

    def _take(self, x, g):
        """[B, K, ...] -> the nodes of group g, [B, n_C, ...]."""
        return x if g.n == self.K else x.index_select(1, g.idx)

    def _pack(self, parts):
        """Per-group spectra [B, n_C, C, ...] -> mask_fn's Y: [B, K, C, ...], or packed [B, M, ...]."""
        if self.channels is None:
            return parts[0]
        p0 = parts[0]
        rest = tuple(p0.shape[3:])
        if len(parts) == 1:
            return p0.view((p0.shape[0], self.M) + rest)
        out = torch.empty((p0.shape[0], self.M) + rest, dtype=p0.dtype, device=p0.device)
        for g, p in zip(self._groups, parts):
            out.index_copy_(1, g.rows, p.view((p.shape[0], g.n * g.C) + rest))
        return out

    def _plane(self, parts, mic):
        """Microphone `mic` of every node, [B, K, ...], from per-group spectra [B, n_C, C, ...]."""
        return self._join([_ref_plane(p, mic) for p in parts])

    def _check_r0_kind(self, R0):
        """R0's tensors (flat), checked for their kind: the pair (R_ss, R_nn) for an int C, a list of K pairs for a
        sequence; ValueError / TypeError before any device work."""
        if self.channels is None:
            if not isinstance(R0, (tuple, list)) or len(R0) != 2:
                raise ValueError("R0 must be the pair (R_ss, R_nn)")
            flat = list(R0)
        else:
            if not isinstance(R0, (tuple, list)) or len(R0) != self.K or \
                    any(not isinstance(p, (tuple, list)) or len(p) != 2 for p in R0):
                raise ValueError("R0 must be a list of K = %d (R_ss, R_nn) pairs, one per node" % self.K)
            flat = [r for p in R0 for r in p]
        for r in flat:
            if not isinstance(r, torch.Tensor) or not r.is_cuda:
                raise TypeError("R0 must hold CUDA tensors (disco_b200 has no CPU path)")
        return flat

    def _check_r0_shapes(self, R0, first, device):
        """R0's dtype, shapes and device: [first, K, F, C, C] per matrix, or [first, F, C_k, C_k] for node k."""
        if self.channels is None:
            R0, want = [R0], [(first, self.K, self.F, self.C, self.C)]
        else:
            want = [(first, self.F, c, c) for c in self.channels]
        for k, (pair, w) in enumerate(zip(R0, want)):
            for r in pair:
                if r.dtype != torch.complex64 or tuple(r.shape) != w or r.device != device:
                    raise ValueError("R0%s matrices must be complex64 [%s] on %s"
                                     % ("" if self.channels is None else "[%d]" % k, ", ".join(map(str, w)), device))

    def _r0_groups(self, R0):
        """R0 -> per group the pair (R_ss, R_nn) [first, n_C, F, C, C] (fresh tensors)."""
        if self.channels is None:
            return [tuple(r.contiguous().clone() for r in R0)]
        return [_group_R0(R0, g.nodes, self.K) for g in self._groups]


class OnlineTangoStream(_Geometry):
    """B streams of K nodes x C microphones (D = C + K - 1 <= 8, or <= 16 with wide=True) that start together and
    advance in lockstep; two-step recursive Tango with the parameters and options of `online_tango`:

        s = OnlineTangoStream(B, K, C, n_fft=512, lambda_cor=0.95, block=8, lag=1)
        out = s.push(y_chunk, mask_fn)     # y_chunk [B, K, C, n] float32 CUDA, any n >= 0
        out = s.flush(mask_fn)             # end of the stream: the last frame and the remaining samples
        st = s.state()                     # or, at any point: save the session (stream_state) ...
        s2 = OnlineTangoStream.from_state(st)   # ... and resume it, here or elsewhere, bit for bit

    mask_fn(t0, Y, z_y, zn) -> (mask_z, mask_w) is called once for each run of newly completed frames [t0, t0 + f),
    after the run's step-1 outputs exist and before any later frame is filtered, with Y [B, K, C, f, F] (the STFT) and
    z_y, zn [B, K, f, F] (step 1).  It returns frame-major float32 masks [B, K, f, F]; mask_w = None means mask_z.
    Precomputed masks are a slice by t0; a causal estimator reads Y, z_y and zn.  A call that completes no frame needs
    no mask_fn.

    Ragged arrays: C may be a sequence of K per-node counts (channels, as in ragged.py; K <= 16, max(C_k) + K - 1 <=
    16, ref_mic a microphone of every node).  Every chunk (and s_chunk, n_chunk) is then packed [B, M, n], M =
    sum(channels), node k on rows off_k .. off_k + C_k - 1; mask_fn's Y is packed [B, M, f, F] (row r: packed
    microphone r); R0 is a list of K pairs (R_ss, R_nn) [B, F, C_k, C_k], as online_tango_ragged takes it; W1 and W2
    are dicts {C: [B, n_C, F, C]} and {C: [B, n_C, F, C + K - 1]} over the nodes of each count (`nodes`).  Every
    other input and output keeps its shape, and the outputs equal online_tango_ragged on the whole signal.  wide=True
    is needed as soon as one count's C_k + K - 1 exceeds 8.  Equal counts ([4, 4, 4, 4]) take packed chunks and
    equal the int-C stream.

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
        B, K = int(B), int(K)
        if B < 1 or K < 1 or (not _is_ragged(C) and int(C) < 1):
            raise ValueError("B, K and C must be positive")
        _check_params(n_fft, block, lambda_cor, lag)
        self._set_geometry(K, C, ref_mic, "stream", wide)
        clean = bool(clean) or vads is not None
        _check_options(filter_type, rank, mask_for_z, clean, vads)
        flat = self._check_r0_kind(R0) if R0 is not None else None
        device = _cuda_device(flat[0].device if device is None and R0 is not None else device, "stream")
        F, H, P = n_fft // 2 + 1, n_fft // 2, int(block)
        self.B, self.F = B, F
        if R0 is not None:
            self._check_r0_shapes(R0, B, device)
        self.n_fft, self.block, self.lag = n_fft, P, int(lag)
        self.lambda_cor, self.mu, self.rank, self.ref_mic = float(lambda_cor), float(mu), rank, int(ref_mic)
        self.filter_type, self.mask_for_z, self.clean = filter_type, mask_for_z, clean
        self.vads = None if vads is None else tuple(vads)
        self.device = device
        self._make_groups(device)
        f32, c64 = dict(dtype=torch.float32, device=device), dict(dtype=torch.complex64, device=device)
        self._oracle1 = "use_oracle_" in mask_for_z
        R0s = self._r0_groups(R0) if R0 is not None else [None] * len(self._groups)
        for g, r0 in zip(self._groups, R0s):
            pair = lambda: [torch.zeros((B, g.n, g.C, n_fft), **f32), torch.zeros((B, g.n, g.C, n_fft), **f32)]
            g.hist = pair()                                             # in, out
            g.hist_sn = (pair(), pair()) if clean else None
            # the open block's spectra, written in place run by run; the clean ones for the 'use_oracle_*' statistics
            g.Yblk = torch.zeros((B, g.n, g.C, P, F), **c64)
            g.SNblk = tuple(torch.zeros((B, g.n, g.C, P, F), **c64) for _ in range(2)) if self._oracle1 else None
            # carried statistics: step 1 from R0; step 2 from R0 for a single node, from zeros otherwise
            g.R1, g.R2 = r0, (r0 if K == 1 else None)
            # solved filters by block index, kept while a later block still uses them; pass-through stand-ins
            g.W1s, g.W2s = {}, {}
            g.pass1 = torch.zeros((B, g.n, 1, F, g.C), **c64)
            g.pass2 = torch.zeros((B, g.n, 1, F, g.D), **c64)
        self._none = torch.empty(self._lead(B) + (0,), **f32)
        # one iSTFT carry per time signal: yf, or the six of TIME_NAMES
        self._carry = torch.zeros((len(TIME_NAMES), B, K, H) if clean else (B, K, H), **f32)
        # the open block over all K nodes: masks and (K > 1) step-1 outputs; z_s and z_n for the exchange modes that
        # read them
        self._m1 = torch.zeros((B, K, P, F), **f32)
        self._m2 = torch.zeros((B, K, P, F), **f32)
        self._zblk = torch.zeros((B, K, P, F), **c64) if K > 1 else None
        self._zsnblk = None
        if K > 1 and mask_for_z in ("compressed", "use_oracle_zs"):
            self._zsnblk = tuple(torch.zeros((B, K, P, F), **c64) for _ in range(2))
        self._L = self._T = self._S = 0
        self._closed = False

    # ---------------------------------------------------------------- state
    def _last_filters(self, step):
        if not self._groups[0].W1s:
            return None
        Ws = {g.C: (g.W1s, g.W2s)[step][max(g.W1s)] for g in self._groups}
        return Ws[self.C] if self.channels is None else Ws

    @property
    def W1(self):
        """Step-1 filters [B, K, F, C] of the last closed block (None before the first); block j's come into force for
        block j + lag.  With per-node counts: {C: [B, n_C, F, C]} over the nodes of each count."""
        return self._last_filters(0)

    @property
    def W2(self):
        """Step-2 filters [B, K, F, D] of the last closed block (None before the first); with per-node counts
        {C: [B, n_C, F, C + K - 1]}."""
        return self._last_filters(1)

    @property
    def _R1(self):
        """The carried step-1 statistics (R_ss, R_nn) of the first group (every node of an int-C stream)."""
        return self._groups[0].R1

    @property
    def _R2(self):
        return self._groups[0].R2

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

    # ---------------------------------------------------------------- saving and resuming
    def state(self, index=None):
        """The session state (stream_state) of all B streams, or of stream `index` alone as a B = 1 state: host copies
        of every tensor, so the stream continues exactly as if it had not been called.  A closed stream raises
        ValueError."""
        if self._closed:
            raise ValueError("the stream is closed (flushed, or an earlier push failed): it has no state to save")
        if index is None:
            take = lambda x, dim=0: stream_state.host(x)
        else:
            if isinstance(index, bool) or not isinstance(index, (int, np.integer)) or not 0 <= index < self.B:
                raise ValueError("index must be a stream in 0..%d, got %r" % (self.B - 1, index))
            i = int(index)
            take = lambda x, dim=0: None if x is None else stream_state.host(x.narrow(dim, i, 1))
        B, J, lag = (self.B if index is None else 1), self._T // self.block, self.lag
        blocks = range(J - min(J, lag), J)

        def filters(g, Ws, d):
            if not blocks:
                return torch.zeros((B, 0, g.n, self.F, d), dtype=torch.complex64)
            return take(torch.stack([Ws[j] for j in blocks], 1))

        groups = []
        for g in self._groups:
            pair = lambda R: None if R is None else [take(R[0]), take(R[1])]
            hs, hn = (take(h[0]) for h in g.hist_sn) if self.clean else (None, None)
            Sb, Nb = (take(b) for b in g.SNblk) if g.SNblk is not None else (None, None)
            groups.append({"C": g.C, "nodes": list(g.nodes), "hist": take(g.hist[0]), "hist_s": hs, "hist_n": hn,
                           "Yblk": take(g.Yblk), "Sblk": Sb, "Nblk": Nb, "R1": pair(g.R1), "R2": pair(g.R2),
                           "W1": filters(g, g.W1s, g.C), "W2": filters(g, g.W2s, g.D)})
        carry = take(self._carry, 1).transpose(0, 1).contiguous() if self.clean else take(self._carry).unsqueeze(1)
        zs, zn = (take(b) for b in self._zsnblk) if self._zsnblk is not None else (None, None)
        return {"version": stream_state.VERSION, "kind": "clean" if self.clean else "plain",
                "n_fft": self.n_fft, "lambda_cor": self.lambda_cor, "block": self.block, "lag": lag, "mu": self.mu,
                "rank": self.rank, "ref_mic": self.ref_mic, "filter_type": self.filter_type,
                "mask_for_z": self.mask_for_z, "clean": self.clean, "vads": self.vads, "wide": self.D > 8,
                "K": self.K, "C": self.C if self.channels is None else None,
                "channels": None if self.channels is None else list(self.channels), "B": B,
                "samples_in": self._L, "frames_out": self._T, "samples_out": self._S, "closed": J,
                "groups": groups, "m1": take(self._m1), "m2": take(self._m2), "zblk": take(self._zblk),
                "zsblk": zs, "znblk": zn, "carry": carry}

    @classmethod
    def from_state(cls, state, device=None):
        """A stream that continues where `state` left off, on `device` (None: the current CUDA device).  A list of
        states of identical options, geometry and counters makes one lockstep stream of B = sum(B_i) streams, in list
        order; its outputs equal those of the streams the states came from when each stream's signals are paired
        among themselves (n_C * C even for every channel-count group, and K even), as for online_tango_ragged's
        batches (DESIGN §4.8).  ValueError for an invalid state or states that do not match, before any device work."""
        st = stream_state.concat(state)
        opts = {k: st[k] for k in ("n_fft", "lambda_cor", "block", "lag", "mu", "rank", "ref_mic")}
        self = cls(st["B"], st["K"], st["C"] if st["channels"] is None else st["channels"], device=device,
                   filter_type=st["filter_type"], mask_for_z=st["mask_for_z"], clean=st["clean"], vads=st["vads"],
                   wide=st["wide"], **opts)
        dev = lambda x: None if x is None else x.to(self.device, copy=True)
        J = st["closed"]
        for g, s in zip(self._groups, st["groups"]):
            g.hist[0].copy_(s["hist"])
            if self.clean:
                g.hist_sn[0][0].copy_(s["hist_s"])
                g.hist_sn[1][0].copy_(s["hist_n"])
            g.Yblk.copy_(s["Yblk"])
            if g.SNblk is not None:
                g.SNblk[0].copy_(s["Sblk"])
                g.SNblk[1].copy_(s["Nblk"])
            g.R1 = None if s["R1"] is None else tuple(dev(r) for r in s["R1"])
            g.R2 = None if s["R2"] is None else tuple(dev(r) for r in s["R2"])
            nw = s["W1"].shape[1]
            g.W1s = {J - nw + i: dev(s["W1"][:, i]).contiguous() for i in range(nw)}
            g.W2s = {J - nw + i: dev(s["W2"][:, i]).contiguous() for i in range(nw)}
        if self.clean:
            self._carry.copy_(st["carry"].transpose(0, 1))
        else:
            self._carry.copy_(st["carry"][:, 0])
        self._m1.copy_(st["m1"])
        self._m2.copy_(st["m2"])
        if self._zblk is not None:
            self._zblk.copy_(st["zblk"])
        if self._zsnblk is not None:
            self._zsnblk[0].copy_(st["zsblk"])
            self._zsnblk[1].copy_(st["znblk"])
        self._L, self._T, self._S = st["samples_in"], st["frames_out"], st["samples_out"]
        return self

    # ---------------------------------------------------------------- public calls
    def push(self, y_chunk, mask_fn=None, *, s_chunk=None, n_chunk=None):
        """Append y_chunk [B, K, C, n] (packed: [B, M, n]) float32 (n >= 0) to every stream, and s_chunk, n_chunk (its
        clean components, shaped like it) to a stream with clean components; returns what became final (class doc)."""
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
        lead = self._lead(self.B)
        if x.dim() != len(lead) + 1 or tuple(x.shape[:-1]) != lead:
            raise ValueError("%s shape %s, expected (%s, n)" % (name, tuple(x.shape), ", ".join(map(str, lead))))
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
        """(W [B, n, 1, F, D], lag argument of filter_sum_blocks) for the frames of block j: the filter of block
        j - lag, or, while that does not exist, the kernel's own pass-through of the reference channel."""
        jw = j - self.lag
        return (stand_in, 1) if jw < 0 else (Ws[jw].unsqueeze(2), 0)

    def _close_block(self, j, nb):
        """Statistics and filters of block j once the masks of its nb frames are in (nb < block: the final, partial
        block, whose recursion step is lambda^nb, as in the whole-signal scan).  The statistics are online_tango's
        for the stream's mask_for_z: the masked scans for 'local', the split scans of [mask Y ; z_rs] and
        [(1 - mask) Y ; z_rn] otherwise, and those of S and N for step 1 under 'use_oracle_*'.  Each stage runs once
        per group, step 2 reading the z of all K nodes."""
        P, lam, n_fft, K, groups = self.block, self.lambda_cor, self.n_fft, self.K, self._groups
        cut = (lambda b: b) if nb == P else (lambda b: None if b is None else b[..., :nb, :].contiguous())
        m1, m2, zb = cut(self._m1), cut(self._m2), cut(self._zblk)
        blk = [(cut(g.Yblk),) + (tuple(cut(b) for b in g.SNblk) if g.SNblk is not None else (None, None))
               for g in groups]
        zsb, znb = (cut(b) for b in self._zsnblk) if self._zsnblk is not None else (None, None)
        # scm_recursive writes fresh matrices, so its output never aliases the carried R0 it reads
        st1 = []
        for g, (Yb, Sb, Nb) in zip(groups, blk):
            if self._oracle1:
                st1.append(_split_scans(Sb, Nb, None, None, None, lam, P, g.R1, n_fft))
            else:
                st1.append(ops.scm_recursive(Yb, self._take(m1, g), None, lam, P, 2, g.R1, n_fft))
        # what the other nodes contribute; a single node has none (online_tango reads its own channels only)
        z_rs = z_rn = None
        if self.mask_for_z != "local" and K > 1:
            kind = self.vads[0] if self.vads is not None else "irm1"
            z_rs, z_rn = _z_for_stats(self.mask_for_z, (kind, kind), zb, m2, zsb, znb,
                                      lambda: (self._plane([b[1] for b in blk], self.ref_mic),
                                               self._plane([b[2] for b in blk], self.ref_mic)))
        st2 = []
        for g, (Yb, _, _) in zip(groups, blk):
            if self.mask_for_z == "local":
                st2.append(ops.scm_recursive(Yb, self._take(m2, g), zb, lam, P, 2, g.R2, n_fft, node_sel=g.sel))
            else:
                st2.append(_split_scans(Yb, Yb, z_rs, z_rn, self._take(m2, g), lam, P, g.R2, n_fft, node_sel=g.sel))
        for g, (Rs1, Rn1), (Rs2, Rn2) in zip(groups, st1, st2):
            g.R1, g.R2 = (Rs1[:, :, 0], Rn1[:, :, 0]), (Rs2[:, :, 0], Rn2[:, :, 0])
            g.W1s[j] = ops.mwf_solve(Rs1, Rn1, self.mu, self.filter_type, self.rank)[0][:, :, 0]
            g.W2s[j] = ops.mwf_solve(Rs2, Rn2, self.mu, self.filter_type, self.rank)[0][:, :, 0]
            for Ws in (g.W1s, g.W2s):
                for old in [i for i in Ws if i < j + 1 - self.lag]:
                    del Ws[old]

    def _advance(self, chunk, sn, L1, T1, S1, mask_fn, final):
        B, K, F, P, n_fft, ref, groups = self.B, self.K, self.F, self.block, self.n_fft, self.ref_mic, self._groups
        T0, S0 = self._T, self._S
        clean = sn is not None
        update = chunk.shape[-1] > 0          # the history moves with every sample that arrives
        xs = self._split(chunk)
        xsn = list(zip(*(self._split(x) for x in sn))) if clean else [None] * len(groups)   # per group: (s, n)
        x_time = torch.empty(((len(TIME_NAMES),) if clean else ()) + (B, K, S1 - S0), dtype=torch.float32,
                             device=self.device)
        names = ["z_y", "zn", "yf"] + (["z_s", "z_n", "sf", "nf"] if clean else []) + \
            (["masks_z", "mask_w"] if self.vads is not None else [])
        parts = []
        if T1 == T0 and update:
            for g, x, xc in zip(groups, xs, xsn):
                ops.stream_stft(g.hist[0], x, L1, T0, 0, n_fft, hist_out=g.hist[1])
                if clean:
                    for x2, (h_in, h_out) in zip(xc, g.hist_sn):
                        ops.stream_stft(h_in, x2, L1, T0, 0, n_fft, hist_out=h_out)
        t = T0
        while t < T1:
            j, slot = divmod(t, P)
            f = min(T1, (j + 1) * P) - t
            last = t + f == T1
            keep = last and update
            Ys, SNs = [], []
            for g, x, xc in zip(groups, xs, xsn):
                Ys.append(ops.stream_stft(g.hist[0], x, L1, t, f, n_fft, hist_out=g.hist[1] if keep else None,
                                          Y_blk=g.Yblk, blk_slot=slot, final=final))
                if clean:
                    # S, N: one transform each, as online_tango takes them (the pairing of signals decides the bits)
                    SNs.append(tuple(ops.stream_stft(h_in, x2, L1, t, f, n_fft, hist_out=h_out if keep else None,
                                                     Y_blk=None if g.SNblk is None else g.SNblk[i], blk_slot=slot,
                                                     final=final)
                                     for i, (x2, (h_in, h_out)) in enumerate(zip(xc, g.hist_sn))))
            Ws = [(self._in_force(g.W1s, g.pass1, j), self._in_force(g.W2s, g.pass2, j)) for g in groups]
            st1 = [ops.filter_sum_blocks(W1, Y, None, P, lg1, True, ref, n_fft) for ((W1, lg1), _), Y in zip(Ws, Ys)]
            z, zn = self._join([a[0] for a in st1]), self._join([a[1] for a in st1])
            yf = self._join([ops.filter_sum_blocks(W2, Y, z if K > 1 else None, P, lg2, True, ref, n_fft,
                                                   node_sel=g.sel)[0]
                             for g, (_, (W2, lg2)), Y in zip(groups, Ws, Ys)])
            if self.vads is None:
                mz, mw = _check_masks(mask_fn(t, self._pack(Ys), z, zn), (B, K, f, F), self.device)
            else:
                # tf_mask is elementwise, so the run's masks are those of the whole signal (tango._clean_masks)
                spectra = lambda c: (self._plane([a[0] for a in SNs], c), self._plane([a[1] for a in SNs], c))
                mz = _step1_mask(self.vads[0], None, lambda: spectra(ref), None, None, n_fft)
                mw = _step2_mask(self.vads, None, mz, lambda: spectra(0), None, n_fft, ref_mic=ref)
            self._m1[:, :, slot:slot + f].copy_(mz)
            self._m2[:, :, slot:slot + f].copy_(mw)
            if K > 1:
                self._zblk[:, :, slot:slot + f].copy_(z)
            part = [z, zn, yf]
            if clean:
                # the diagnostics of online_tango: W1 on S, N; W2 on [S_own ; z_s], [N_own ; z_n]
                zsn = [tuple(ops.filter_sum_blocks(W1, X, None, P, lg1, True, ref, n_fft)[0] for X in sng)
                       for ((W1, lg1), _), sng in zip(Ws, SNs)]
                z_s, z_n = self._join([a[0] for a in zsn]), self._join([a[1] for a in zsn])
                sfn = [tuple(ops.filter_sum_blocks(W2, X, Zx if K > 1 else None, P, lg2, True, ref, n_fft,
                                                   node_sel=g.sel)[0] for X, Zx in zip(sng, (z_s, z_n)))
                       for g, (_, (W2, lg2)), sng in zip(groups, Ws, SNs)]
                sf, nf = self._join([a[0] for a in sfn]), self._join([a[1] for a in sfn])
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
            for g in groups:
                g.hist.reverse()
                if clean:
                    for h in g.hist_sn:
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


class OnlineTangoPool(_Geometry):
    """S slots, each an independent online Tango stream of K nodes x C microphones that opens, advances and closes on
    its own; the parameters are those of OnlineTangoStream, filter_type and the exchange modes that need no clean
    components ('local', 'distant', 'previous') included, and one pool has one geometry (D = C + K - 1 <= 16):

        pool = OnlineTangoPool(S, K, C, n_fft=512, lambda_cor=0.95, block=8, lag=1)
        pool.open(slots, R0=None)        # R0 = (R_ss, R_nn) complex64 [len(slots), K, F, C, C], or None
        out = pool.push(y, n, mask_fn)   # y [S, K, C, n_max] float32 CUDA; slot s gets y[s, ..., :n[s]]
        out = pool.close(slots, mask_fn) # the last frame (reflected at the end), the partial block, the last samples
        pool.filters(slot)               # (W1 [K, F, C], W2 [K, F, D]) of the slot's last closed block, or None
        st = pool.export(slot, release=False)   # the slot's session (stream_state); release=True frees the slot
        pool.restore(slot, st)           # a free slot resumes a session of this pool's options and geometry

    For every slot, its outputs concatenated over the calls from open to close equal, value for value, those of
    OnlineTangoStream(1, K, C) with the same options fed the same samples (hence online_tango on the slot's whole
    signal and ops.istft of its yf), with the masks mask_fn returned -- whatever the other slots do, the slot's index,
    and the cut of its samples into pushes.  A slot's K C signals are paired into transforms inside the slot, as the single stream pairs them.

    Ragged arrays: C may be a sequence of K per-node counts, as for OnlineTangoStream.  y is then packed [S, M, n_max];
    mask_fn's Y is packed [S, M, f_max, F]; open takes R0 as a list of K pairs [len(slots), F, C_k, C_k]; filters
    returns the dicts ({C: [n_C, F, C]}, {C: [n_C, F, C + K - 1]}) over the nodes of each count (`nodes`).  A slot's
    signals pair inside each of its groups, so it equals OnlineTangoStream(1, K, channels).

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
        S, K = int(S), int(K)
        if S < 1 or K < 1 or (not _is_ragged(C) and int(C) < 1):
            raise ValueError("S, K and C must be positive")
        _check_params(n_fft, block, lambda_cor, lag)
        self._set_geometry(K, C, ref_mic, "pool", True)
        _check_options(filter_type, rank, mask_for_z, False, None)
        if S > 65535:
            raise ValueError("at most 65535 slots")
        device = _cuda_device(device, "pool")
        self.S, self.F = S, n_fft // 2 + 1
        self.n_fft, self.block, self.lag = n_fft, int(block), int(lag)
        self.lambda_cor, self.mu, self.rank, self.ref_mic = float(lambda_cor), float(mu), rank, int(ref_mic)
        self.filter_type, self.mask_for_z = filter_type, mask_for_z
        self.device = device
        self._make_groups(device)
        # host state per slot
        self._open = np.zeros(S, dtype=bool)
        self._L = np.zeros(S, dtype=np.int64)          # samples in
        self._T = np.zeros(S, dtype=np.int64)          # frames out
        self._S = np.zeros(S, dtype=np.int64)          # time samples out
        self._par = np.zeros(S, dtype=np.int64)        # which history buffer holds the slot's last n_fft samples
        self._nclosed = np.zeros(S, dtype=np.int64)    # closed blocks
        self._seeded = np.zeros(S, dtype=bool)         # opened with R0: the carried matrices exist before a block
        self._bufs = False

    def _alloc(self):
        """Device state, allocated on the first open."""
        if self._bufs:
            return
        S, K, F, P, N, dev = self.S, self.K, self.F, self.block, self.n_fft, self.device
        f32, c64 = dict(dtype=torch.float32, device=dev), dict(dtype=torch.complex64, device=dev)
        self._carry = torch.zeros((S, K, N // 2), **f32)
        # the open block of every slot over all K nodes: masks and (K > 1) step-1 outputs
        self._m1 = torch.zeros((S, K, P, F), **f32)
        self._m2 = torch.zeros((S, K, P, F), **f32)
        self._zblk = torch.zeros((S, K, P, F), **c64) if K > 1 else None
        for g in self._groups:
            C, D, n = g.C, g.D, g.n
            g.hist = torch.zeros((2, S, n, C, N), **f32)
            g.Yblk = torch.zeros((S, n, C, P, F), **c64)      # the open block's spectra
            # carried statistics (zeros stand for "none yet": the scan's R_(-1) is 0 either way)
            g.R1 = (torch.zeros((S, n, F, C, C), **c64), torch.zeros((S, n, F, C, C), **c64))
            g.R2 = (torch.zeros((S, n, F, D, D), **c64), torch.zeros((S, n, F, D, D), **c64))
            # ring of the last lag + 1 filters: block j's at j % (lag + 1).  Entries of blocks before the first hold
            # the pass-through of the reference channel, stored as (e_ref, -0) so that the kernel's conjugate is
            # exactly the weight vector of filter_sum_blocks' own pass-through.
            g.W1 = torch.zeros((S, self.lag + 1, n, F, C), **c64)
            g.W2 = torch.zeros((S, self.lag + 1, n, F, D), **c64)
            g.pass_ = []
            for d in (C, D):
                re = torch.zeros((n, F, d), **f32)
                re[..., self.ref_mic] = 1.0
                g.pass_.append(torch.complex(re, torch.full_like(re, -0.0)))
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
        its first; kept after close until the slot is opened again.  With per-node counts: ({C: [n_C, F, C]},
        {C: [n_C, F, C + K - 1]})."""
        s = int(self._slot_list([slot])[0])
        if self._nclosed[s] == 0:
            return None
        pos = int((self._nclosed[s] - 1) % (self.lag + 1))
        Ws = {g.C: (g.W1[s, pos].clone(), g.W2[s, pos].clone()) for g in self._groups}
        if self.channels is None:
            return Ws[self.C]
        return {C: w[0] for C, w in Ws.items()}, {C: w[1] for C, w in Ws.items()}

    # ---------------------------------------------------------------- public calls
    def open(self, slots, R0=None):
        """Open free slots: every slot starts a new stream (history, block buffers, filters and iSTFT carry reset; the
        carried matrices from R0, or zeros).  R0 = (R_ss, R_nn), complex64 [len(slots), K, F, C, C] (per-node counts:
        a list of K pairs [len(slots), F, C_k, C_k])."""
        idx = self._slot_list(slots)
        if self._open[idx].any():
            raise ValueError("slot %d is already open" % int(idx[self._open[idx]][0]))
        if R0 is not None:
            self._check_r0_kind(R0)
            self._check_r0_shapes(R0, len(idx), self.device)
        if len(idx) == 0:
            return
        self._alloc()
        K = self.K
        i = torch.from_numpy(idx).to(self.device)
        self._carry[i] = 0
        for buf in (self._m1, self._m2, self._zblk):
            if buf is not None:
                buf[i] = 0
        R0s = self._r0_groups(R0) if R0 is not None else [None] * len(self._groups)
        for g, r0 in zip(self._groups, R0s):
            g.hist[:, i] = 0
            g.Yblk[i] = 0
            for w in range(2):
                g.R1[w][i] = 0 if r0 is None else r0[w]
                g.R2[w][i] = r0[w] if (r0 is not None and K == 1) else 0   # step 2 of a single node starts from R0
            g.W1[i] = g.pass_[0]
            g.W2[i] = g.pass_[1]
        self._open[idx] = True
        self._seeded[idx] = R0 is not None
        for a in (self._L, self._T, self._S, self._par, self._nclosed):
            a[idx] = 0

    def push(self, y, n, mask_fn):
        """Append y[s, ..., :n[s]] to slot s (y [S, K, C, n_max], packed [S, M, n_max], float32 CUDA; n host ints,
        0 <= n[s] <= n_max, and 0 for free slots); returns what became final (class doc)."""
        if not isinstance(y, torch.Tensor):
            raise TypeError("y must be a CUDA tensor (disco_b200 has no CPU path)")
        lead = self._lead(self.S)
        if y.dim() != len(lead) + 1 or tuple(y.shape[:-1]) != lead:
            raise ValueError("y shape %s, expected (%s, n_max)" % (tuple(y.shape), ", ".join(map(str, lead))))
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
        chunk = torch.empty(self._lead(self.S) + (0,), dtype=torch.float32, device=self.device)
        out = self._run(chunk, np.zeros(self.S, dtype=np.int64), self._L.copy(), T1, S1, final, mask_fn)
        self._open[idx] = False
        return out

    # ---------------------------------------------------------------- saving and moving sessions
    def _one_slot(self, slot):
        idx = self._slot_list([slot])
        if len(idx) != 1:
            raise ValueError("one slot, got %r" % (slot,))
        return int(idx[0])

    def export(self, slot, release=False):
        """The session state (stream_state) of open slot `slot`: a B = 1 state in the format of
        OnlineTangoStream.state(index), as host copies.  release=True frees the slot without emitting its tail; the
        session lives on in the state."""
        s = self._one_slot(slot)
        if not self._open[s]:
            raise ValueError("slot %d is not open" % s)
        take = lambda x: stream_state.host(x[s:s + 1])
        J, lag = int(self._nclosed[s]), self.lag
        # the ring holds block j's filters at j % (lag + 1); the state keeps blocks J - nw .. J - 1
        pos = torch.tensor([j % (lag + 1) for j in range(J - min(J, lag), J)], dtype=torch.int64)
        groups = []
        for g in self._groups:
            R1 = None if J == 0 and not self._seeded[s] else [take(g.R1[0]), take(g.R1[1])]
            R2 = None if J == 0 and (self.K > 1 or not self._seeded[s]) else [take(g.R2[0]), take(g.R2[1])]
            groups.append({"C": g.C, "nodes": list(g.nodes), "hist": take(g.hist[int(self._par[s])]),
                           "hist_s": None, "hist_n": None, "Yblk": take(g.Yblk), "Sblk": None, "Nblk": None,
                           "R1": R1, "R2": R2, "W1": take(g.W1)[:, pos], "W2": take(g.W2)[:, pos]})
        state = {"version": stream_state.VERSION, "kind": "plain",
                 "n_fft": self.n_fft, "lambda_cor": self.lambda_cor, "block": self.block, "lag": lag, "mu": self.mu,
                 "rank": self.rank, "ref_mic": self.ref_mic, "filter_type": self.filter_type,
                 "mask_for_z": self.mask_for_z, "clean": False, "vads": None, "wide": self.D > 8,
                 "K": self.K, "C": self.C if self.channels is None else None,
                 "channels": None if self.channels is None else list(self.channels), "B": 1,
                 "samples_in": int(self._L[s]), "frames_out": int(self._T[s]), "samples_out": int(self._S[s]),
                 "closed": J, "groups": groups, "m1": take(self._m1), "m2": take(self._m2),
                 "zblk": None if self._zblk is None else take(self._zblk), "zsblk": None, "znblk": None,
                 "carry": take(self._carry).unsqueeze(1)}
        if release:
            self._open[s] = False
        return state

    def restore(self, slot, state):
        """Open free slot `slot` from a B = 1 session state (stream_state): its later outputs from push and close
        equal those the exporting stream or slot would have produced.  The state's options and geometry must be the
        pool's, and it cannot hold clean components; ValueError before any change otherwise.  The state's tensors
        are copied to the pool's device."""
        s = self._one_slot(slot)
        if self._open[s]:
            raise ValueError("slot %d is already open" % s)
        stream_state.check(state)
        if state["B"] != 1:
            raise ValueError("session state: B = %d: a slot takes one stream (OnlineTangoStream.state(index))"
                             % state["B"])
        if state["clean"]:
            raise ValueError("session state: clean components cannot go into a pool (its slots take none)")
        mine = {"n_fft": self.n_fft, "lambda_cor": self.lambda_cor, "block": self.block, "lag": self.lag,
                "mu": self.mu, "rank": self.rank, "ref_mic": self.ref_mic, "filter_type": self.filter_type,
                "mask_for_z": self.mask_for_z, "K": self.K, "C": self.C if self.channels is None else None,
                "channels": None if self.channels is None else list(self.channels)}
        for k, v in mine.items():
            if state[k] != v:
                raise ValueError("session state: %s is %r, the pool's %r" % (k, state[k], v))
        self._alloc()
        J, lag = state["closed"], self.lag
        for g, st in zip(self._groups, state["groups"]):
            g.hist[0, s].copy_(st["hist"][0])
            g.Yblk[s].copy_(st["Yblk"][0])
            for R, Rst in ((g.R1, st["R1"]), (g.R2, st["R2"])):
                for w in range(2):
                    if Rst is None:
                        R[w][s] = 0                      # "none yet": the scan's R_(-1) is 0 either way
                    else:
                        R[w][s].copy_(Rst[w][0])
            g.W1[s] = g.pass_[0]
            g.W2[s] = g.pass_[1]
            nw = st["W1"].shape[1]
            for i in range(nw):
                g.W1[s, (J - nw + i) % (lag + 1)].copy_(st["W1"][0, i])
                g.W2[s, (J - nw + i) % (lag + 1)].copy_(st["W2"][0, i])
        self._m1[s].copy_(state["m1"][0])
        self._m2[s].copy_(state["m2"][0])
        if self._zblk is not None:
            self._zblk[s].copy_(state["zblk"][0])
        self._carry[s].copy_(state["carry"][0, 0])
        self._open[s] = True
        self._seeded[s] = state["groups"][0]["R1"] is not None
        self._L[s], self._T[s], self._S[s] = state["samples_in"], state["frames_out"], state["samples_out"]
        self._par[s], self._nclosed[s] = 0, J

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
        masks of its nb[s] frames are in (nb < block: the final, partial block, whose recursion step is lambda^nb).
        Each stage runs once per group, step 2 reading the z of all K nodes."""
        P, lam, n_fft, groups = self.block, self.lambda_cor, self.n_fft, self._groups
        m1, m2 = self._m1[ci], self._m2[ci]
        zb = self._zblk[ci] if self.K > 1 else None
        Ybs = [g.Yblk[ci] for g in groups]
        st1 = [ops.scm_recursive(Yb, self._take(m1, g), None, lam, P, 2, (g.R1[0][ci], g.R1[1][ci]), n_fft,
                                 frames=nb) for g, Yb in zip(groups, Ybs)]
        z_rs = z_rn = None
        if self.mask_for_z != "local" and zb is not None:
            z_rs, z_rn = _z_for_stats(self.mask_for_z, None, zb, m2, None, None, None)
        st2 = []
        for g, Yb in zip(groups, Ybs):
            R2 = (g.R2[0][ci], g.R2[1][ci])
            if self.mask_for_z == "local":
                st2.append(ops.scm_recursive(Yb, self._take(m2, g), zb, lam, P, 2, R2, n_fft, node_sel=g.sel,
                                             frames=nb))
            else:
                st2.append(_split_scans(Yb, Yb, z_rs, z_rn, self._take(m2, g), lam, P, R2, n_fft, frames=nb,
                                        node_sel=g.sel))
        pos = None
        for g, (Rs1, Rn1), (Rs2, Rn2) in zip(groups, st1, st2):
            W1 = ops.mwf_solve(Rs1, Rn1, self.mu, self.filter_type, self.rank)[0][:, :, 0]
            W2 = ops.mwf_solve(Rs2, Rn2, self.mu, self.filter_type, self.rank)[0][:, :, 0]
            for R, new in ((g.R1, (Rs1, Rn1)), (g.R2, (Rs2, Rn2))):
                R[0][ci] = new[0][:, :, 0]
                R[1][ci] = new[1][:, :, 0]
            if pos is None:
                pos = torch.from_numpy(self._nclosed[cl] % (self.lag + 1)).to(self.device)
            g.W1[ci, pos] = W1
            g.W2[ci, pos] = W2
        self._nclosed[cl] += 1

    def _advance(self, chunk, n, L1, T1, S1, final, mask_fn):
        S, K, F, P, lag, n_fft, ref, dev = (self.S, self.K, self.F, self.block, self.lag, self.n_fft, self.ref_mic,
                                            self.device)
        groups = self._groups
        T0, S0 = self._T.copy(), self._S.copy()
        frames, samples = T1 - T0, S1 - S0
        starts, runs = pool_rounds(T0, T1, P)
        c64 = dict(dtype=torch.complex64, device=dev)
        f_call = int(frames.max())
        out = [torch.zeros((S, K, f_call, F), **c64) for _ in range(3)]        # z_y, zn, yf
        yf_time = torch.zeros((S, K, int(samples.max())), dtype=torch.float32, device=dev)
        write = n > 0
        xs = self._split(chunk)
        stft_rec = np.zeros((S, len(ops.STFT_SLOT_FIELDS)), dtype=np.int64)
        stft_rec[:, 0], stft_rec[:, 1], stft_rec[:, 5], stft_rec[:, 6] = L1, n, final, self._par
        istft_rec = np.zeros((S, len(ops.ISTFT_SLOT_FIELDS)), dtype=np.int64)
        istft_rec[:, 2], istft_rec[:, 4] = L1, S0
        if len(runs) == 0 and write.any():       # no frame completes: only the history moves
            stft_rec[:, 2], stft_rec[:, 7] = T0, write
            for g, x in zip(groups, xs):
                ops.stream_stft_slots(g.hist, x, stft_rec, 0, n_fft)
        for r in range(len(runs)):
            t0, nr = starts[r], runs[r]
            act = np.nonzero(nr)[0]
            fr, f = nr[act], int(nr.max())
            blk = np.where(nr > 0, t0 % P, 0)
            stft_rec[:, 2], stft_rec[:, 3], stft_rec[:, 4], stft_rec[:, 7] = t0, nr, blk, write if r == 0 else 0
            Ys = [ops.stream_stft_slots(g.hist, x, stft_rec, f, n_fft, Y_blk=g.Yblk) for g, x in zip(groups, xs)]
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
            Yas = Ys if every else [Y[ai] for Y in Ys]
            # step 1 and step 2 with the filter in force, W_(j - lag) (the pass-through stand-in before the first)
            st1 = [ops.filter_sum_blocks(g.W1[ai, pi].unsqueeze(2), Ya, None, P, 0, True, ref, n_fft, frames=fr)
                   for g, Ya in zip(groups, Yas)]
            z, zn = self._join([a[0] for a in st1]), self._join([a[1] for a in st1])
            yf = self._join([ops.filter_sum_blocks(g.W2[ai, pi].unsqueeze(2), Ya, z if K > 1 else None, P, 0, True,
                                                   ref, n_fft, node_sel=g.sel, frames=fr)[0]
                             for g, Ya in zip(groups, Yas)])
            if every:
                zf, znf, yff = z, zn, yf
            else:
                zf, znf, yff = (torch.zeros((S, K, f, F), **c64) for _ in range(3))
                zf[ai], znf[ai], yff[ai] = z, zn, yf
            mz, mw = _check_masks(mask_fn(t0.copy(), nr.copy(), self._pack(Ys), zf, znf), (S, K, f, F), dev)
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
