"""Batched Tango on ragged arrays: nodes with different microphone counts (reference tango.py:252-290).

Layout.  A batch of B utterances of one array of K nodes with channels = (C_0, ..., C_{K-1}) microphones is packed:
y [B, M, L] float32 on the device, M = sum(channels), node k's microphones being rows off_k .. off_k + C_k - 1 with
off_k = sum(channels[:k]).  The clean components s, n use the same layout; masks are [B, K, T, F] as everywhere.

Every step runs once per distinct channel count C on the nodes that have it (CatArgs, csrc/kernels.h): the group's
rows are gathered into [B, n_C, C, L], step 1 runs on them (tango_step1 / online.online_mwf), the compressed signals
of all K nodes are assembled with index_copy, and step 2 runs on the group with node_sel so that its kernels read
the z of every other node (tango_step2 / ops.scm_recursive, ops.filter_sum_blocks).  Between launches there are only
gathers, index_copy and views: no arithmetic on spectra or signals and no host synchronisation.

A group's STFT is one call over its [B, n_C, C, L] signals, which the transform pairs as signals 2p, 2p + 1 of that
call (DESIGN §5).  So when n_C * C is even for every group, every utterance's signals are paired as in a lone run
(B = 1), and the online outputs of an utterance equal its lone run bit for bit.

The outputs are those of tango.tango_batched / online.online_tango, [B, K, ...] over all K nodes, so that
post.to_time and post.tango_scores take them unchanged.
"""
import numpy as np
import torch

from . import ops
from .online import _live_blocks, _online_mwf_split, online_mwf
from .tango import (_check_sources, _frame_clip, _step1_mask, _step2_mask, _uneven_lengths, _z_for_stats, tango_step1,
                    tango_step2)

MAX_CHANNELS = 16          # the step-2 kernels take C + K - 1 <= 16 channels (and so K <= 16 nodes)


class _Layout:
    """The packed layout of `channels`: K, the offsets, and the nodes of each channel count (ascending counts).  M:
    the packed rows the caller holds, or None where no rows are at hand yet (a stream, before its first chunk)."""

    def __init__(self, channels, M, ref_mic):
        if isinstance(channels, (str, bytes, torch.Tensor)) or not hasattr(channels, "__len__") or len(channels) == 0:
            raise TypeError("channels must be a non-empty sequence of microphone counts, one per node")
        for c in channels:
            if isinstance(c, (bool, np.bool_)) or not isinstance(c, (int, np.integer)):
                raise TypeError("channels must be integers, got %r" % (c,))
            if c < 1:
                raise ValueError("every node needs at least one microphone, got %r" % (channels,))
        self.channels = [int(c) for c in channels]
        self.K = len(self.channels)
        if M is not None and sum(self.channels) != M:
            raise ValueError("channels %r sum to %d, y holds %d rows" % (self.channels, sum(self.channels), M))
        if self.K > MAX_CHANNELS:
            raise NotImplementedError("at most %d nodes, got %d" % (MAX_CHANNELS, self.K))
        D = max(self.channels) + self.K - 1
        if D > MAX_CHANNELS:
            raise NotImplementedError("C + K - 1 must be <= %d, got %d" % (MAX_CHANNELS, D))
        if isinstance(ref_mic, (bool, np.bool_)) or not isinstance(ref_mic, (int, np.integer)):
            raise TypeError("ref_mic must be an integer")
        if not 0 <= ref_mic < min(self.channels):
            raise ValueError("ref_mic %d is not a microphone of every node (channels %r)" % (ref_mic, self.channels))
        self.offsets = np.concatenate([[0], np.cumsum(self.channels)[:-1]]).astype(np.int64)
        groups = {}
        for k, c in enumerate(self.channels):
            groups.setdefault(c, []).append(k)
        self.groups = sorted(groups.items())                   # [(C, [nodes])]
        self._idx = {}

    def node_index(self, C, device):
        """The nodes of count C as a device index (built once per call and device)."""
        key = ("nodes", C, str(device))
        if key not in self._idx:
            self._idx[key] = torch.tensor(dict(self.groups)[C], dtype=torch.int64, device=device)
        return self._idx[key]

    def rows(self, C, device):
        """The packed rows of the nodes of count C, node-major: gathering them gives [B, n_C * C, L]."""
        key = ("rows", C, str(device))
        if key not in self._idx:
            r = [int(self.offsets[k]) + c for k in dict(self.groups)[C] for c in range(C)]
            self._idx[key] = torch.tensor(r, dtype=torch.int64, device=device)
        return self._idx[key]

    def mic_rows(self, mic, device):
        """Row of microphone `mic` of every node: gathering them gives [B, K, L]."""
        key = ("mic", mic, str(device))
        if key not in self._idx:
            self._idx[key] = torch.from_numpy(self.offsets + mic).to(device)
        return self._idx[key]

    def gather(self, x, C):
        """x [B, M, L] -> the signals of the nodes of count C, [B, n_C, C, L] (contiguous)."""
        n = len(dict(self.groups)[C])
        return x.index_select(1, self.rows(C, x.device)).view(x.shape[0], n, C, x.shape[-1])


def _check_packed(y, s, n, masks, lay_args):
    """The argument checks of the packed inputs, lay_args = (channels, ref_mic, n_fft, filter_type, rank); returns the
    _Layout.  Nothing here touches the device."""
    if not isinstance(y, torch.Tensor) or y.dim() != 3 or y.dtype != torch.float32:
        raise ValueError("y must be a float32 tensor [B, M, L] (packed microphones)")
    for name, a in (("s", s), ("n", n)):
        if a is not None and (not isinstance(a, torch.Tensor) or tuple(a.shape) != tuple(y.shape)
                              or a.dtype != torch.float32):
            raise ValueError("%s must be a float32 tensor shaped like y %s" % (name, tuple(y.shape)))
    lay = _Layout(lay_args[0], y.shape[1], lay_args[1])
    ops._filter_args(*lay_args[3:])                          # AttributeError for an unknown filter type
    if masks is not None:
        B, L, n_fft = y.shape[0], y.shape[2], lay_args[2]
        want = (B, lay.K, ops.n_frames(L, n_fft), n_fft // 2 + 1)
        for m in masks:
            if isinstance(m, torch.Tensor) and tuple(m.shape) != want:
                raise ValueError("masks must be [B, K, T, F] = %s, got %s" % (want, tuple(m.shape)))
    return lay


def _new(B, K, T, F, dtype, device):
    return torch.empty((B, K, T, F), dtype=dtype, device=device)


def _put(dst, idx, src):
    """dst[:, idx] = src along the node axis (one index_copy)."""
    dst.index_copy_(1, idx, src)


def _masks(lay, y, s, masks, vads, ref_mic, n_fft, lens, spectra):
    """(mask_z, mask_w) [B, K, T, F] of all K nodes.  masks=None: vads[0] of microphone ref_mic and vads[1] of
    microphone 0 from the clean spectra, as tango._clean_masks builds them; spectra(mic) -> (S, N) [B, K, T, F] of that
    microphone of every node, taken from the per-group transforms."""
    if masks is not None:
        mask_z, mask_w = masks
        return mask_z, (mask_z if mask_w is None else mask_w)
    mic = lambda x, c: x.index_select(1, lay.mic_rows(c, x.device))
    mask_z = _step1_mask(vads[0], None, lambda: spectra(ref_mic), mic(s, ref_mic), None, n_fft, lens)
    return mask_z, _step2_mask(vads, None, mask_z, lambda: spectra(0), mic(s, 0), n_fft, ref_mic=ref_mic, lengths=lens)


class _Spectra:
    """Per-group clean spectra S, N [B, n_C, C, T, F] and, on demand, one microphone of them over all K nodes."""

    def __init__(self, lay, s, n, lens, n_fft, B, T, F):
        stft = (lambda a: ops.stft(a, n_fft)) if lens is None else (lambda a: ops.stft_lengths(a, lens, n_fft))
        self.lay, self.shape, self.dev = lay, (B, lay.K, T, F), s.device
        self.SN = {C: (stft(lay.gather(s, C)), stft(lay.gather(n, C))) for C, _ in lay.groups}
        self._mic = {}

    def mic(self, c):
        if c not in self._mic:
            S0, N0 = _new(*self.shape, torch.complex64, self.dev), _new(*self.shape, torch.complex64, self.dev)
            for C, _ in self.lay.groups:
                idx = self.lay.node_index(C, self.dev)
                S, N = self.SN[C]
                _put(S0, idx, S[:, :, c])
                _put(N0, idx, N[:, :, c])
            self._mic[c] = (S0, N0)
        return self._mic[c]


def _mic0_spectra(lay, Y):
    """Y {C: [B, n_C, C, T, F]} -> microphone 0 of every node, [B, K, 1, T, F] (what a step-2 mask estimator reads)."""
    C0 = lay.groups[0][0]
    B, _, _, T, F = Y[C0].shape
    out = torch.empty((B, lay.K, 1, T, F), dtype=torch.complex64, device=Y[C0].device)
    for C, _ in lay.groups:
        out.index_copy_(1, lay.node_index(C, out.device), Y[C][:, :, :1])
    return out


def _callable_mask_w(fn, lay, Y, z_y, zn, clip):
    m = fn(_mic0_spectra(lay, Y), z_y, zn)
    return m if clip is None else clip(m)


def tango_ragged(y, channels, s=None, n=None, masks=None, vads=("irm1", "irm1"), mask_for_z="local", n_fft=512, mu=1.0,
                 filter_type="gevd", rank=1, ref_mic=0, out_layout="FT", diagnostics=True, lengths=None):
    """Two-step Tango on a batch of ragged arrays in the packed layout (module docstring).

    y [B, M, L] float32 CUDA tensor, channels = microphones per node (sum M); s, n [B, M, L] or None; masks =
    (mask_z, mask_w) [B, K, T, F] frame-major or None; mask_w may be None (mask_z) or a callable
    mask_w(Y0, z_y, zn) -> [B, K, T, F] called after step 1, with Y0 [B, K, 1, T, F] the spectra of microphone 0 of
    every node (the one channel all nodes have) and z_y, zn [B, K, T, F].  Every other argument is tango_batched's,
    with its meaning; ref_mic must be a microphone of every node.  Returns tango_batched's dict: yf, z_y, zn,
    masks_z, mask_w and, with s, n and diagnostics, sf, nf, z_s, z_n, all [B, K, F, T] ('FT') or [B, K, T, F] ('TF').
    Argument errors are raised before any device work."""
    _check_sources(masks, s, n, vads, mask_for_z)
    lay = _check_packed(y, s, n, masks, (channels, ref_mic, n_fft, filter_type, rank))
    ft = ops._layout(out_layout) == ops.FT
    B, _, L = y.shape
    K, dev = lay.K, y.device
    T, F = ops.n_frames(L, n_fft), n_fft // 2 + 1
    lens = _uneven_lengths(lengths, B, L, n_fft)
    clip = None if lens is None else _frame_clip(lens, T, n_fft, dev)
    have_sn = s is not None and n is not None
    sp = None
    if have_sn and (masks is None or diagnostics or "use_oracle_" in mask_for_z or mask_for_z == "compressed"):
        sp = _Spectra(lay, s, n, lens, n_fft, B, T, F)
    mask_z, mask_w = _masks(lay, y, s, masks, vads, ref_mic, n_fft, lens, None if sp is None else sp.mic)
    if clip is not None:
        mz = clip(mask_z)
        mask_w = mz if mask_w is mask_z else (mask_w if callable(mask_w) else clip(mask_w))
        mask_z = mz
    # ---- step 1, once per channel count
    osn = "use_oracle_" in mask_for_z
    want_zs = have_sn and (diagnostics or mask_for_z in ("compressed", "use_oracle_zs"))
    Z, ZN = _new(B, K, T, F, torch.complex64, dev), _new(B, K, T, F, torch.complex64, dev)
    Zs = Zn = None
    if want_zs:
        Zs, Zn = _new(B, K, T, F, torch.complex64, dev), _new(B, K, T, F, torch.complex64, dev)
    Y = {}
    for C, nodes in lay.groups:
        idx = lay.node_index(C, dev)
        mz = mask_z.index_select(1, idx)
        st1 = tango_step1(lay.gather(y, C), mz, n_fft, mu, filter_type, rank, ref_mic,
                          oracle_sn=sp.SN[C] if osn else None, lengths=lens)
        Y[C] = st1["Y"]
        _put(Z, idx, st1["z_y"])
        _put(ZN, idx, st1["zn"])
        if want_zs:
            S, N = sp.SN[C]
            W1 = st1["W1"]
            _put(Zs, idx, ops.filter_sum(W1, S, None, conj=True, n_fft=n_fft))
            _put(Zn, idx, ops.filter_sum(W1, N, None, conj=True, n_fft=n_fft))
    if callable(mask_w):
        mask_w = _callable_mask_w(mask_w, lay, Y, Z, ZN, clip)
    z_rs, z_rn = _z_for_stats(mask_for_z, vads, Z, mask_w, Zs, Zn, lambda: sp.mic(ref_mic), clip)
    # ---- step 2, once per channel count, reading the z of all K nodes
    oshape = (B, K, F, T) if ft else (B, K, T, F)
    out = {"yf": torch.empty(oshape, dtype=torch.complex64, device=dev)}
    diag = have_sn and diagnostics
    if diag:
        out["sf"] = torch.empty(oshape, dtype=torch.complex64, device=dev)
        out["nf"] = torch.empty(oshape, dtype=torch.complex64, device=dev)
    for C, nodes in lay.groups:
        idx = lay.node_index(C, dev)
        yf, W2 = tango_step2(Y[C], Z, mask_w.index_select(1, idx), n_fft, mu, filter_type, rank, out_layout,
                             node_sel=nodes, z_rs=z_rs, z_rn=z_rn)
        _put(out["yf"], idx, yf)
        if diag:
            S, N = sp.SN[C]
            _put(out["sf"], idx, ops.filter_sum(W2, S, Zs, conj=True, n_fft=n_fft, out_layout=out_layout,
                                                node_sel=nodes))
            _put(out["nf"], idx, ops.filter_sum(W2, N, Zn, conj=True, n_fft=n_fft, out_layout=out_layout,
                                                node_sel=nodes))
    conv = ops.transpose_last2 if ft else (lambda a: a)
    out["z_y"], out["zn"] = conv(Z), conv(ZN)
    if diag:
        out["z_s"], out["z_n"] = conv(Zs), conv(Zn)
    out["masks_z"] = conv(mask_z)
    out["mask_w"] = out["masks_z"] if mask_w is mask_z else conv(mask_w)
    return out


def _online_step2(Y, Xs, Xn, Z, Zs, Zn, mask, nodes, lambda_cor, block, lag, mu, filter_type, rank, ref, n_fft,
                  frames):
    """Step 2 of online Tango on the nodes `nodes` (Y [B, n, C, T, F]), reading the z of all K nodes (Z [B, K, T, F]):
    online.online_mwf (Xs = None: the masked scans of [Y ; Z]) or online._online_mwf_split (the unweighted scans of
    [mask Xs ; Zs] and [(1 - mask) Xn ; Zn], filters on [Y ; Z]), on the same kernels with node_sel.
    Returns dict(z, zn, W)."""
    if Xs is None:
        Rss, Rnn = ops.scm_recursive(Y, mask, Z, lambda_cor, block, 2, None, n_fft, node_sel=nodes, frames=frames)
    else:
        Xs, Xn = ops.apply_mask(Xs, mask, False), ops.apply_mask(Xn, mask, True)
        Rss, _ = ops.scm_recursive(Xs, None, Zs, lambda_cor, block, 2, None, n_fft, node_sel=nodes, frames=frames)
        Rnn, _ = ops.scm_recursive(Xn, None, Zn, lambda_cor, block, 2, None, n_fft, node_sel=nodes, frames=frames)
    W, _ = ops.mwf_solve(Rss, Rnn, mu, filter_type, rank)
    W = _live_blocks(W, frames, Y.shape[3], block)
    z, zn = ops.filter_sum_blocks(W, Y, Z, block, lag, True, ref, n_fft, node_sel=nodes, frames=frames)
    return {"z": z, "zn": zn, "W": W}


def _group_R0(R0, nodes, K):
    """R0 = K pairs (R_ss, R_nn) [B, F, C_k, C_k] -> the pair of the nodes `nodes`, [B, n, F, C, C] each."""
    return tuple(torch.stack([R0[k][i] for k in nodes], 1) for i in (0, 1))


def _check_R0(R0, lay, B, F):
    if R0 is None:
        return
    if not isinstance(R0, (list, tuple)) or len(R0) != lay.K:
        raise ValueError("R0 must be a list of K = %d (R_ss, R_nn) pairs" % lay.K)
    for k, pair in enumerate(R0):
        C = lay.channels[k]
        if len(pair) != 2 or any(not isinstance(r, torch.Tensor) or tuple(r.shape) != (B, F, C, C)
                                 or r.dtype != torch.complex64 for r in pair):
            raise ValueError("R0[%d] must be two complex64 [B, F, C, C] = %s tensors" % (k, (B, F, C, C)))


def online_tango_ragged(y, channels, masks=None, lambda_cor=0.95, block=8, lag=1, mu=1.0, rank=1, ref_mic=0, n_fft=512,
                        R0=None, lengths=None, *, s=None, n=None, vads=("irm1", "irm1"), mask_for_z="local",
                        filter_type="gevd", diagnostics=True):
    """online.online_tango on a batch of ragged arrays in the packed layout (module docstring).

    y, s, n [B, M, L]; channels, masks and a callable mask_w as tango_ragged takes them; R0: None or a list of K pairs
    (R_ss, R_nn) [B, F, C_k, C_k] seeding step 1 of node k (step 2 of a multi-node array starts from zeros).  Every
    other argument is online_tango's, with its meaning.  Returns online_tango's outputs [B, K, T, F] (yf, z_y, zn;
    with s, n and diagnostics z_s, z_n, sf, nf; with masks=None masks_z, mask_w) and, per channel count C, the block
    filters of its nodes: W1[C] [B, n_C, J, F, C], W2[C] [B, n_C, J, F, C + K - 1] and nodes[C], their node indices.
    Argument errors are raised before any device work."""
    _check_sources(masks, s, n, vads, mask_for_z)
    lay = _check_packed(y, s, n, masks, (channels, ref_mic, n_fft, filter_type, rank))
    B, _, L = y.shape
    K, dev = lay.K, y.device
    T, F = ops.n_frames(L, n_fft), n_fft // 2 + 1
    _check_R0(R0, lay, B, F)
    lens = _uneven_lengths(lengths, B, L, n_fft)
    frames = clip = None
    if lens is not None:
        frames, clip = ops.n_frames(lens, n_fft), _frame_clip(lens, T, n_fft, dev)
    stft = (lambda a: ops.stft(a, n_fft)) if lens is None else (lambda a: ops.stft_lengths(a, lens, n_fft))
    Y = {C: stft(lay.gather(y, C)) for C, _ in lay.groups}
    have_sn = s is not None and n is not None
    sp = None
    if have_sn and (masks is None or diagnostics or "use_oracle_" in mask_for_z or mask_for_z == "compressed"):
        sp = _Spectra(lay, s, n, lens, n_fft, B, T, F)
    mask_z, mask_w = _masks(lay, y, s, masks, vads, ref_mic, n_fft, lens, None if sp is None else sp.mic)
    if clip is not None:
        mz = clip(mask_z)
        mask_w = mz if mask_w is mask_z else (mask_w if callable(mask_w) else clip(mask_w))
        mask_z = mz
    opts = (lambda_cor, block, lag, mu, filter_type, rank, ref_mic)
    # ---- step 1, once per channel count (independent single-node problems)
    want_zs = have_sn and (diagnostics or mask_for_z in ("compressed", "use_oracle_zs"))
    Z, ZN = _new(B, K, T, F, torch.complex64, dev), _new(B, K, T, F, torch.complex64, dev)
    Zs = Zn = None
    if want_zs:
        Zs, Zn = _new(B, K, T, F, torch.complex64, dev), _new(B, K, T, F, torch.complex64, dev)
    W1 = {}
    for C, nodes in lay.groups:
        idx = lay.node_index(C, dev)
        r0 = None if R0 is None else _group_R0(R0, nodes, K)
        if "use_oracle_" in mask_for_z:
            s1 = _online_mwf_split(Y[C], *sp.SN[C], None, None, None, None, *opts, r0, n_fft, frames)
        else:
            s1 = online_mwf(Y[C], mask_z.index_select(1, idx), None, *opts, 2, r0, n_fft, frames)
        W1[C] = s1["W"]
        _put(Z, idx, s1["z"])
        _put(ZN, idx, s1["zn"])
        if want_zs:
            S, N = sp.SN[C]
            _put(Zs, idx, ops.filter_sum_blocks(W1[C], S, None, block, lag, True, ref_mic, n_fft, frames=frames)[0])
            _put(Zn, idx, ops.filter_sum_blocks(W1[C], N, None, block, lag, True, ref_mic, n_fft, frames=frames)[0])
    if callable(mask_w):
        mask_w = _callable_mask_w(mask_w, lay, Y, Z, ZN, clip)
    z_rs, z_rn = _z_for_stats(mask_for_z, vads, Z, mask_w, Zs, Zn, lambda: sp.mic(ref_mic), clip)
    # ---- step 2, once per channel count, reading the z of all K nodes
    out = {"yf": _new(B, K, T, F, torch.complex64, dev), "z_y": Z, "zn": ZN}
    diag = have_sn and diagnostics
    if diag:
        out["sf"], out["nf"] = _new(B, K, T, F, torch.complex64, dev), _new(B, K, T, F, torch.complex64, dev)
    W2 = {}
    for C, nodes in lay.groups:
        idx = lay.node_index(C, dev)
        mw = mask_w.index_select(1, idx)
        if K == 1:
            # a single node has no other nodes: step 2 reads its own channels only and starts from R0 like step 1
            r0 = None if R0 is None else _group_R0(R0, nodes, K)
            if z_rs is None:
                s2 = online_mwf(Y[C], mw, None, *opts, 2, r0, n_fft, frames)
            else:
                s2 = _online_mwf_split(Y[C], Y[C], Y[C], None, None, None, mw, *opts, r0, n_fft, frames)
        elif z_rs is None:
            s2 = _online_step2(Y[C], None, None, Z, None, None, mw, nodes, *opts, n_fft, frames)
        else:
            s2 = _online_step2(Y[C], Y[C], Y[C], Z, z_rs, z_rn, mw, nodes, *opts, n_fft, frames)
        W2[C] = s2["W"]
        _put(out["yf"], idx, s2["z"])
        if diag:
            S, N = sp.SN[C]
            Zsel = (None, None) if K == 1 else (Zs, Zn)
            sel = None if K == 1 else nodes
            _put(out["sf"], idx, ops.filter_sum_blocks(W2[C], S, Zsel[0], block, lag, True, ref_mic, n_fft,
                                                       node_sel=sel, frames=frames)[0])
            _put(out["nf"], idx, ops.filter_sum_blocks(W2[C], N, Zsel[1], block, lag, True, ref_mic, n_fft,
                                                       node_sel=sel, frames=frames)[0])
    if diag:
        out["z_s"], out["z_n"] = Zs, Zn
    if masks is None:
        out["masks_z"], out["mask_w"] = mask_z, mask_w
    out["W1"], out["W2"] = W1, W2
    out["nodes"] = {C: list(nodes) for C, nodes in lay.groups}
    return out
