"""Tensor-level operators of the MWF path: thin wrappers that hand torch CUDA tensors (device
memory + current stream) to the C ABI of libdisco_b200.so.  PyTorch is plumbing here: all
arithmetic happens in the hand-written kernels.

Layouts: spectra are frame-major ``[..., T, F]`` complex64; ``layout='FT'`` arguments select the
reference's NumPy layout ``[..., F, T]`` for masks / final outputs (SURVEY.md §8b op table).
"""
import collections
import ctypes
import math

import numpy as np
import torch

from . import _lib

TF, FT = 0, 1
MASK_KINDS = {"irm": 0, "ibm": 1, "iam": 2}
FILTER_TYPES = {"gevd": 0, "r1-mwf": 1, "mwf": 2}


def _layout(layout):
    if layout in (TF, "TF", "tf"):
        return TF
    if layout in (FT, "FT", "ft"):
        return FT
    raise ValueError("layout must be 'TF' or 'FT'")


def _stream():
    """Current stream of the CURRENT device; every public op below runs under the device of its operands
    (see `_on_device`), so this is the stream of the tensors' device."""
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _on_device(fn):
    """Run an op with the device of its tensor operands current: the library keeps per-device tables
    (cudaGetDevice) and launches on the current stream, so operands on another device than the current one
    would otherwise be dereferenced by kernels running on the wrong GPU.  Mixed devices are rejected."""
    import functools

    @functools.wraps(fn)
    def wrapper(*args, **kw):
        dev = None
        stack = list(args) + list(kw.values())
        while stack:
            a = stack.pop()
            if isinstance(a, (tuple, list)):
                stack.extend(a)
            elif isinstance(a, torch.Tensor) and a.is_cuda:
                if dev is None:
                    dev = a.device
                elif a.device != dev:
                    raise ValueError("%s: operands live on different devices (%s, %s)" % (fn.__name__, dev, a.device))
        if dev is None or dev.index == torch.cuda.current_device():
            return fn(*args, **kw)
        with torch.cuda.device(dev):
            return fn(*args, **kw)
    return wrapper


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _need(t, dtype, name):
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise TypeError("%s must be a CUDA tensor (disco_b200 has no CPU path)" % name)
    if t.dtype != dtype:
        raise TypeError("%s must be %s, got %s" % (name, dtype, t.dtype))
    if not t.is_contiguous():
        raise ValueError("%s must be contiguous" % name)
    return t


def _bins(F, n_fft, name):
    """Spectra handed to a kernel hold n_fft / 2 + 1 bins: the library derives F from n_fft alone."""
    if F != n_fft // 2 + 1:
        raise ValueError("%s has %d bins, n_fft=%d needs %d" % (name, F, n_fft, n_fft // 2 + 1))


# What a workspace of stft_scm(keep_partials=True) / stft_scm2 was written with: its consumers read the per-segment
# partial sums with the launch plan of these sizes AND of the reserved-SM setting current when they run.
WorkspacePlan = collections.namedtuple("WorkspacePlan", "G C L n_fft n_set reserved_sms")
_reserved_sms = 0     # the value last given to set_reserved_sms (the library's setting is process-wide)


def _workspace(ws, G, C, L, n_fft, n_set):
    """Check that `ws` is a workspace written for (G, C, L, n_fft, n_set) under the current reserved-SM setting and
    holds the bytes its consumers read."""
    _need(ws, torch.float32, "ws")
    plan = getattr(ws, "disco_plan", None)
    if not isinstance(plan, WorkspacePlan):
        raise ValueError("ws is not a workspace returned by stft_scm(keep_partials=True) or stft_scm2")
    want = WorkspacePlan(int(G), int(C), int(L), int(n_fft), int(n_set), _reserved_sms)
    if plan != want:
        raise ValueError("workspace written for %s, read as %s" % (tuple(plan), tuple(want)))
    lib = _lib.load()
    size = lib.disco_stft_scm_workspace if n_set == 1 else lib.disco_stft_scm2_workspace
    need = size(int(G), int(C), int(L), int(n_fft))
    if ws.numel() * ws.element_size() < need:
        raise ValueError("workspace holds %d bytes, %d needed" % (ws.numel() * ws.element_size(), need))


def n_frames(length, n_fft=512):
    """1 + L // hop (reference tango.py:287)."""
    return 1 + length // (n_fft // 2)


def init(n_fft=512):
    """Create the per-device FFT tables now (required before CUDA-graph capture)."""
    _lib.check(_lib.load().disco_init(int(n_fft)))


@_on_device
def stft(x, n_fft=512):
    """x [..., L] float32 -> Y [..., T, F] complex64 (librosa center/reflect/periodic-Hann semantics)."""
    _need(x, torch.float32, "x")
    if x.dim() < 1:
        raise ValueError("x must be [..., samples]")
    L = x.shape[-1]
    n_sig = x.numel() // L
    T, F = n_frames(L, n_fft), n_fft // 2 + 1
    Y = torch.empty(x.shape[:-1] + (T, F), dtype=torch.complex64, device=x.device)
    _lib.check(_lib.load().disco_stft(_ptr(x), _ptr(Y), n_sig, L, n_fft, _stream()))
    return Y


@_on_device
def stft_scm(x, mask, n_fft=512, mask_layout="TF", keep_partials=False):
    """Fused STFT + masked SCM.  x [G, C, L] float32, mask [G, T, F] (or [G, F, T]) float32
    -> Y [G, C, T, F] complex64, Rss, Rnn [G, F, C, C] complex64.
    keep_partials=True returns (Y, workspace) instead: the SCMs stay as per-segment partial sums that
    mwf_solve_workspace() consumes directly (one launch fewer)."""
    _need(x, torch.float32, "x")
    _need(mask, torch.float32, "mask")
    if x.dim() != 3:
        raise ValueError("x must be [groups, channels, samples]")
    G, C, L = x.shape
    T, F = n_frames(L, n_fft), n_fft // 2 + 1
    lib = _lib.load()
    if not lib.disco_stft_scm_supported(n_fft, C, 1):
        raise NotImplementedError("fused STFT+SCM: %d channels at n_fft=%d (use stft + masked_scm)" % (C, n_fft))
    lay = _layout(mask_layout)
    want = (G, T, F) if lay == TF else (G, F, T)
    if tuple(mask.shape) != want:
        raise ValueError("mask shape %s, expected %s" % (tuple(mask.shape), want))
    Y = torch.empty((G, C, T, F), dtype=torch.complex64, device=x.device)
    ws_bytes = lib.disco_stft_scm_workspace(G, C, L, n_fft)
    ws = torch.empty(max(ws_bytes, 16) // 4, dtype=torch.float32, device=x.device)
    if keep_partials:
        _lib.check(lib.disco_stft_scm(_ptr(x), _ptr(mask), lay, _ptr(Y), None, None, G, C, L, n_fft,
                                      _ptr(ws), ws_bytes, _stream()))
        ws.disco_plan = WorkspacePlan(G, C, L, int(n_fft), 1, _reserved_sms)
        return Y, ws
    Rss = torch.empty((G, F, C, C), dtype=torch.complex64, device=x.device)
    Rnn = torch.empty_like(Rss)
    _lib.check(lib.disco_stft_scm(_ptr(x), _ptr(mask), lay, _ptr(Y), _ptr(Rss), _ptr(Rnn), G, C, L, n_fft,
                                  _ptr(ws), ws_bytes, _stream()))
    return Y, Rss, Rnn


@_on_device
def mwf_solve_workspace(ws, G, C, L, n_fft=512, mu=1.0, type="gevd", rank=1, want_scm=False):
    """mwf_solve on the SCMs a preceding stft_scm(..., keep_partials=True) left in `ws`.
    Returns W, t1 [G, F, C] (and Rss, Rnn [G, F, C, C] when want_scm)."""
    ftype, r = _filter_args(type, rank)
    _workspace(ws, G, C, L, n_fft, 1)
    F = n_fft // 2 + 1
    W = torch.empty((G, F, C), dtype=torch.complex64, device=ws.device)
    T1 = torch.empty_like(W)
    Rss = Rnn = None
    if want_scm:
        Rss = torch.empty((G, F, C, C), dtype=torch.complex64, device=ws.device)
        Rnn = torch.empty_like(Rss)
    _lib.check(_lib.load().disco_mwf_solve_workspace(_ptr(ws), _ptr(W), _ptr(T1), _ptr(Rss), _ptr(Rnn), G, C, L, n_fft,
                                                     ftype, r, float(mu), _stream()))
    return (W, T1, Rss, Rnn) if want_scm else (W, T1)


def set_reserved_sms(n):
    """Leave n SMs free of the persistent fused STFT+SCM kernel (room for a concurrent NCCL collective).  A workspace
    is consumed under the setting it was written with (the consumers refuse it otherwise).  The setting is tracked
    here: a direct call of the library's disco_set_reserved_sms bypasses it, and a workspace written and consumed
    after such a call is then only checked for its sizes and byte count."""
    global _reserved_sms
    _lib.check(_lib.load().disco_set_reserved_sms(int(n)))
    _reserved_sms = int(n)


def stft_scm_supported(n_fft, C, n_mask=1):
    """Whether the fused STFT+SCM kernel covers (n_fft, channels per group, number of masks)."""
    return bool(_lib.load().disco_stft_scm_supported(int(n_fft), int(C), int(n_mask)))


@_on_device
def stft_scm2(x, mask_a, mask_b, n_fft=512, mask_layout="TF", want_Y=True):
    """Fused STFT + the masked SCMs under TWO masks in one pass (single-node arrays: step-1 and step-2
    statistics are taken over the same Y, reference tango.py:357-364 and :431-440 with K = 1).
    x [G, C, L], masks [G, T, F] (or [G, F, T]) -> Y [G, C, T, F], workspace (partial sums of both sets,
    consumed by mwf_solve_workspace2 / scm_from_workspace).  want_Y=False stores no spectrum and returns
    (None, workspace); the workspace is the same bit for bit."""
    _need(x, torch.float32, "x")
    _need(mask_a, torch.float32, "mask_a")
    _need(mask_b, torch.float32, "mask_b")
    if x.dim() != 3:
        raise ValueError("x must be [groups, channels, samples]")
    G, C, L = x.shape
    T, F = n_frames(L, n_fft), n_fft // 2 + 1
    lib = _lib.load()
    if not lib.disco_stft_scm_supported(n_fft, C, 2):
        raise NotImplementedError("two-mask fused STFT+SCM: %d channels at n_fft=%d" % (C, n_fft))
    lay = _layout(mask_layout)
    want = (G, T, F) if lay == TF else (G, F, T)
    if tuple(mask_a.shape) != want or tuple(mask_b.shape) != want:
        raise ValueError("mask shapes %s / %s, expected %s" % (tuple(mask_a.shape), tuple(mask_b.shape), want))
    Y = torch.empty((G, C, T, F), dtype=torch.complex64, device=x.device) if want_Y else None
    ws_bytes = lib.disco_stft_scm2_workspace(G, C, L, n_fft)
    ws = torch.empty(max(ws_bytes, 16) // 4, dtype=torch.float32, device=x.device)
    _lib.check(lib.disco_stft_scm2(_ptr(x), _ptr(mask_a), _ptr(mask_b), lay, _ptr(Y), G, C, L, n_fft, _ptr(ws),
                                   ws_bytes, _stream()))
    ws.disco_plan = WorkspacePlan(G, C, L, int(n_fft), 2, _reserved_sms)
    return Y, ws


@_on_device
def scm_from_workspace(ws, G, C, L, n_fft=512, n_set=1, set=0):
    """Rss, Rnn [G, F, C, C] of mask set `set` from the partial sums a fused STFT+SCM call left in `ws`."""
    _workspace(ws, G, C, L, n_fft, n_set)
    F = n_fft // 2 + 1
    Rss = torch.empty((G, F, C, C), dtype=torch.complex64, device=ws.device)
    Rnn = torch.empty_like(Rss)
    _lib.check(_lib.load().disco_scm_from_workspace(_ptr(ws), int(n_set), int(set), _ptr(Rss), _ptr(Rnn), G, C, L,
                                                    n_fft, _stream()))
    return Rss, Rnn


@_on_device
def mwf_solve_workspace2(ws, G, C, L, n_fft=512, mu=1.0, type="gevd", rank=1):
    """Both filter sets of a stft_scm2 workspace in one launch: W, t1 [2, G, F, C] (0: mask_a, 1: mask_b)."""
    ftype, r = _filter_args(type, rank)
    _workspace(ws, G, C, L, n_fft, 2)
    F = n_fft // 2 + 1
    W = torch.empty((2, G, F, C), dtype=torch.complex64, device=ws.device)
    T1 = torch.empty_like(W)
    _lib.check(_lib.load().disco_mwf_solve_workspace2(_ptr(ws), _ptr(W), _ptr(T1), G, C, L, n_fft,
                                                      ftype, r, float(mu), _stream()))
    return W, T1


@_on_device
def filter_dual(W1, W2, Y, ref=0, n_fft=512, out_layout="TF", want_zn=True):
    """Single-node groups: z = w1^H y, zn = y[ref] - z and yf = w2^H y in ONE pass over Y (reference
    tango.py:369-376 and :445-450 with K = 1).  W1, W2 [..., F, C], Y [..., C, T, F] -> z, zn, yf
    [..., T, F] (or [..., F, T])."""
    _need(W1, torch.complex64, "W1")
    _need(W2, torch.complex64, "W2")
    _need(Y, torch.complex64, "Y")
    if Y.dim() < 3:
        raise ValueError("Y must be [..., C, T, F]")
    C, T, F = Y.shape[-3:]
    _bins(F, n_fft, "Y")
    lead = tuple(Y.shape[:-3])
    G = Y.numel() // (C * T * F)
    if tuple(W1.shape) != lead + (F, C) or tuple(W2.shape) != lead + (F, C):
        raise ValueError("W1 / W2 shape %s / %s, expected %s" % (tuple(W1.shape), tuple(W2.shape), lead + (F, C)))
    lay = _layout(out_layout)
    shape = lead + ((T, F) if lay == TF else (F, T))
    z = torch.empty(shape, dtype=torch.complex64, device=Y.device)
    zn = torch.empty_like(z) if want_zn else None
    yf = torch.empty_like(z)
    _lib.check(_lib.load().disco_filter_dual(_ptr(W1), _ptr(W2), _ptr(Y), _ptr(z), _ptr(zn), _ptr(yf), int(ref), lay,
                                             G, C, T, n_fft, _stream()))
    return z, zn, yf


@_on_device
def stft_filter_dual(x, W1, W2, ref=0, n_fft=512, out_layout="TF", want_zn=True):
    """filter_dual(W1, W2, stft(x)) without the spectrum in memory: the fused STFT kernel transforms the time signals
    again and applies z = w1^H y, zn = y[ref] - z and yf = w2^H y per (frame, bin).  x [G, C, L] float32, W1, W2
    [G, F, C] -> z, zn, yf [G, T, F] (or [G, F, T], written in that layout by the kernel)."""
    _need(x, torch.float32, "x")
    _need(W1, torch.complex64, "W1")
    _need(W2, torch.complex64, "W2")
    if x.dim() != 3:
        raise ValueError("x must be [groups, channels, samples]")
    G, C, L = x.shape
    T, F = n_frames(L, n_fft), n_fft // 2 + 1
    lib = _lib.load()
    if not lib.disco_stft_scm_supported(n_fft, C, 2):
        raise NotImplementedError("fused STFT+filter: %d channels at n_fft=%d" % (C, n_fft))
    if tuple(W1.shape) != (G, F, C) or tuple(W2.shape) != (G, F, C):
        raise ValueError("W1 / W2 shape %s / %s, expected %s" % (tuple(W1.shape), tuple(W2.shape), (G, F, C)))
    lay = _layout(out_layout)
    z = torch.empty((G, T, F) if lay == TF else (G, F, T), dtype=torch.complex64, device=x.device)
    zn = torch.empty_like(z) if want_zn else None
    yf = torch.empty_like(z)
    _lib.check(lib.disco_stft_filter_dual(_ptr(x), _ptr(W1), _ptr(W2), _ptr(z), _ptr(zn), _ptr(yf), int(ref), lay,
                                          G, C, L, n_fft, _stream()))
    return z, zn, yf


@_on_device
def tf_mask(S, N, type="irm1", bin_thr=0.0):
    """Oracle mask (reference dnn/utils.py:44-71) on device, float32.  Same shape as S."""
    _need(S, torch.complex64, "S")
    _need(N, torch.complex64, "N")
    if S.shape != N.shape:
        raise AssertionError("Input spectrograms should have the same shape.")   # sigproc_utils.py:71
    kind = type[:-1] if len(type) > 1 else ""
    if kind not in MASK_KINDS or not type[-1].isdigit():
        raise ValueError('Unknown mask type. Should be "irmX", "ibmX" or "iamX"')
    M = torch.empty(S.shape, dtype=torch.float32, device=S.device)
    _lib.check(_lib.load().disco_tf_mask(_ptr(S), _ptr(N), _ptr(M), S.numel(), MASK_KINDS[kind], int(type[-1]),
                                         float(bin_thr), _stream()))
    return M


def _cat_geometry(y_shape, z_shape=None, node_sel=None, z_layout="BK"):
    """Launch geometry of the concatenated channels [Y ; z of the other nodes] (CatArgs, csrc/kernels.h), checked
    here because the library only sees pointers.  y_shape = (B, Ksel, C, T, F); z_shape = (B, K, T, F) with
    z_layout 'BK', node-major (K, B, T, F) with 'KB' (what an all-gather over node-owning ranks delivers,
    disco_b200/dist.py), or None: no exchange, every (b, k) is an independent single-node problem.  node_sel: the
    nodes Y holds (None = all K).  Returns n_utt, K, sel (ctypes int array or None), n_sel, z_layout flag."""
    if len(y_shape) != 5:
        raise ValueError("Y shape %s, expected [B, Ksel, C, T, F]" % (tuple(y_shape),))
    B, Ks, C, T, F = y_shape
    if z_shape is None:
        return B * Ks, 1, None, 1, 0
    if z_layout not in ("BK", "KB"):
        raise ValueError("z_layout must be 'BK' or 'KB'")
    K = z_shape[1 if z_layout == "BK" else 0] if len(z_shape) == 4 else 0
    want = (B, K, T, F) if z_layout == "BK" else (K, B, T, F)
    if tuple(z_shape) != want:
        raise ValueError("Z shape %s, expected %s" % (tuple(z_shape), want))
    sel, n_sel = None, K
    if node_sel is not None:
        sel, n_sel = (ctypes.c_int * len(node_sel))(*[int(v) for v in node_sel]), len(node_sel)
    if Ks != n_sel:
        raise ValueError("Y holds %d nodes, selection has %d" % (Ks, n_sel))
    return B, K, sel, n_sel, (0 if z_layout == "BK" else 1)


def _cat_args(Y, Z, node_sel, n_fft, z_layout="BK"):
    """_cat_geometry of the tensors Y (complex64, [B, Ksel, C, T, F], F = n_fft / 2 + 1) and Z (complex64 or None)."""
    _need(Y, torch.complex64, "Y")
    if Z is not None:
        _need(Z, torch.complex64, "Z")
    if Y.dim() == 5:
        _bins(Y.shape[-1], n_fft, "Y")
    return _cat_geometry(tuple(Y.shape), None if Z is None else tuple(Z.shape), node_sel, z_layout)


def _filter_args(type, rank):
    """Library code of an intern_filter type and the eigenpair count (0 = all, for rank 'full' / 'Full' / None)."""
    if type not in FILTER_TYPES:
        raise AttributeError("Unknown filter reference")       # internal_formulas.py:79
    return FILTER_TYPES[type], 0 if rank in ("full", "Full", None) else int(rank)


@_on_device
def masked_scm(Y, mask, Z=None, n_fft=512, mask_layout="TF", node_sel=None, z_layout="BK"):
    """Y [B, Ksel, C, T, F], Z [B, K, T, F] (or [K, B, T, F] with z_layout='KB') or None (K = 1),
    mask [B, Ksel, T, F] / [B, Ksel, F, T] or None
    -> Rss, Rnn [B, Ksel, F, D, D], D = C + K - 1 (own mics, then z of the other nodes)."""
    n_utt, K, sel, n_sel, zl = _cat_args(Y, Z, node_sel, n_fft, z_layout)
    B, Ks, C, T, F = Y.shape
    lay = _layout(mask_layout)
    if mask is not None:
        _need(mask, torch.float32, "mask")
        want = (B, Ks, T, F) if lay == TF else (B, Ks, F, T)
        if tuple(mask.shape) != want:
            raise ValueError("mask shape %s, expected %s" % (tuple(mask.shape), want))
    D = C + K - 1
    Rss = torch.empty((B, Ks, F, D, D), dtype=torch.complex64, device=Y.device)
    Rnn = torch.empty_like(Rss)
    _lib.check(_lib.load().disco_masked_scm(_ptr(Y), _ptr(Z), _ptr(mask), lay, _ptr(Rss), _ptr(Rnn), n_utt, K, C, T,
                                            n_fft, sel, n_sel, zl, _stream()))
    return Rss, Rnn


@_on_device
def filter_sum_scm(W1, Y, mask, ref=0, n_fft=512, mask_layout="TF"):
    """Single-node groups (no exchange): z = w1^H y, zn = y[ref] - z AND the masked SCMs of Y under `mask`
    in one pass over Y.  W1 [..., F, C], Y [..., C, T, F], mask [..., T, F] (or [..., F, T]).
    Returns z, zn [..., T, F], Rss, Rnn [..., F, C, C]."""
    _need(W1, torch.complex64, "W1")
    _need(Y, torch.complex64, "Y")
    _need(mask, torch.float32, "mask")
    if Y.dim() < 3:
        raise ValueError("Y must be [..., C, T, F]")
    C, T, F = Y.shape[-3:]
    _bins(F, n_fft, "Y")
    lead = Y.shape[:-3]
    G = Y.numel() // (C * T * F)
    lay = _layout(mask_layout)
    if tuple(W1.shape) != tuple(lead) + (F, C):
        raise ValueError("W1 shape %s, expected %s" % (tuple(W1.shape), tuple(lead) + (F, C)))
    want = tuple(lead) + ((T, F) if lay == TF else (F, T))
    if tuple(mask.shape) != want:
        raise ValueError("mask shape %s, expected %s" % (tuple(mask.shape), want))
    z = torch.empty(lead + (T, F), dtype=torch.complex64, device=Y.device)
    zn = torch.empty_like(z)
    Rss = torch.empty(lead + (F, C, C), dtype=torch.complex64, device=Y.device)
    Rnn = torch.empty_like(Rss)
    _lib.check(_lib.load().disco_filter_sum_scm(_ptr(W1), _ptr(Y), _ptr(mask), lay, _ptr(z), _ptr(zn), int(ref),
                                                _ptr(Rss), _ptr(Rnn), G, C, T, n_fft, _stream()))
    return z, zn, Rss, Rnn


def tango_mid_supported(C, K):
    return bool(_lib.load().disco_tango_mid_supported(int(C), int(K)))


@_on_device
def tango_mid(W1, Y, mask_w, ref=0, n_fft=512):
    """Multi-node arrays: z, zn of every node AND the step-2 SCMs of every node in one pass over Y.
    W1 [B, K, F, C], Y [B, K, C, T, F], mask_w [B, K, T, F] -> z, zn [B, K, T, F], Rss, Rnn [B, K, F, D, D]."""
    _need(W1, torch.complex64, "W1")
    _need(Y, torch.complex64, "Y")
    _need(mask_w, torch.float32, "mask_w")
    if Y.dim() != 5:
        raise ValueError("Y must be [B, K, C, T, F]")
    B, K, C, T, F = Y.shape
    _bins(F, n_fft, "Y")
    D = C + K - 1
    if tuple(W1.shape) != (B, K, F, C) or tuple(mask_w.shape) != (B, K, T, F):
        raise ValueError("W1 %s / mask_w %s, expected %s / %s" % (tuple(W1.shape), tuple(mask_w.shape), (B, K, F, C),
                                                                  (B, K, T, F)))
    z = torch.empty((B, K, T, F), dtype=torch.complex64, device=Y.device)
    zn = torch.empty_like(z)
    Rss = torch.empty((B, K, F, D, D), dtype=torch.complex64, device=Y.device)
    Rnn = torch.empty_like(Rss)
    _lib.check(_lib.load().disco_tango_mid(_ptr(W1), _ptr(Y), _ptr(mask_w), _ptr(z), _ptr(zn), int(ref), _ptr(Rss),
                                           _ptr(Rnn), B, K, C, T, n_fft, _stream()))
    return z, zn, Rss, Rnn


@_on_device
def mwf_solve(Rss, Rnn, mu=1.0, type="gevd", rank=1):
    """Batched intern_filter (reference internal_formulas.py:31-81).  Rss, Rnn [..., D, D] complex64
    -> W [..., D], t1 [..., D] complex64.  rank 'full'/'Full'/None -> all eigenpairs."""
    _need(Rss, torch.complex64, "Rss")
    _need(Rnn, torch.complex64, "Rnn")
    ftype, r = _filter_args(type, rank)
    if Rss.dim() < 2 or Rss.shape[-1] != Rss.shape[-2] or Rnn.shape != Rss.shape:
        raise ValueError("Rss %s / Rnn %s, expected two [..., D, D]" % (tuple(Rss.shape), tuple(Rnn.shape)))
    D = Rss.shape[-1]
    n_mat = Rss.numel() // (D * D)
    W = torch.empty(Rss.shape[:-1], dtype=torch.complex64, device=Rss.device)
    T1 = torch.empty_like(W)
    _lib.check(_lib.load().disco_mwf_solve(_ptr(Rss), _ptr(Rnn), _ptr(W), _ptr(T1), n_mat, D, ftype, r,
                                           float(mu), _stream()))
    return W, T1


@_on_device
def filter_sum(W, Y, Z=None, conj=True, ref=None, n_fft=512, out_layout="TF", node_sel=None, z_layout="BK"):
    """out = w^H x (conj=True) or w^T x over the concatenated channels [Y ; z of other nodes].
    W [B, Ksel, F, D]; Z [B, K, T, F] (or [K, B, T, F] with z_layout='KB');
    returns out (and resid = x[ref] - out when ref is given), [B, Ksel, T, F] or [.., F, T]."""
    _need(W, torch.complex64, "W")
    n_utt, K, sel, n_sel, zl = _cat_args(Y, Z, node_sel, n_fft, z_layout)
    B, Ks, C, T, F = Y.shape
    D = C + K - 1
    if tuple(W.shape) != (B, Ks, F, D):
        raise ValueError("W shape %s, expected %s" % (tuple(W.shape), (B, Ks, F, D)))
    lay = _layout(out_layout)
    shape = (B, Ks, T, F) if lay == TF else (B, Ks, F, T)
    out = torch.empty(shape, dtype=torch.complex64, device=Y.device)
    resid = torch.empty_like(out) if ref is not None else None
    _lib.check(_lib.load().disco_filter_sum(_ptr(W), 1 if conj else 0, _ptr(Y), _ptr(Z), _ptr(out), _ptr(resid),
                                            0 if ref is None else int(ref), lay, n_utt, K, C, T, n_fft, sel, n_sel,
                                            zl, _stream()))
    return (out, resid) if ref is not None else out


@_on_device
def istft(Y, length, n_fft=512):
    """Y [..., T, F] complex64 -> x [..., length] float32 (librosa istft semantics, center=True)."""
    _need(Y, torch.complex64, "Y")
    T, F = Y.shape[-2:]
    if F != n_fft // 2 + 1:
        raise ValueError("last dimension must be n_fft/2 + 1 bins")
    n_sig = Y.numel() // (T * F)
    x = torch.empty(Y.shape[:-2] + (int(length),), dtype=torch.float32, device=Y.device)
    _lib.check(_lib.load().disco_istft(_ptr(Y), _ptr(x), n_sig, T, int(length), n_fft, _stream()))
    return x


def signal_lengths(lengths, lead, L, lo=0):
    """Per-signal lengths of a batch [*lead, L]: `lengths` (sequence, NumPy array or tensor of integers) covers the
    leading axes lead[:m] and is repeated over the rest (e.g. one length per utterance of [B, K, C, L]).  Every
    length must satisfy lo < length <= L.  Returns the flattened lengths as a host int32 NumPy array."""
    import numpy as np
    if isinstance(lengths, torch.Tensor):
        if lengths.is_floating_point() or lengths.is_complex():
            raise TypeError("lengths must be integers, got %s" % lengths.dtype)
        lengths = lengths.detach().cpu().numpy()
    arr = np.asarray(lengths)
    if arr.dtype.kind not in "iu":
        raise TypeError("lengths must be integers, got %s" % arr.dtype)
    lead = tuple(int(v) for v in lead)
    if arr.ndim > len(lead) or tuple(arr.shape) != lead[:arr.ndim]:
        raise ValueError("lengths shape %s does not match the leading axes %s" % (tuple(arr.shape), lead))
    if arr.size and (int(arr.min()) <= lo or int(arr.max()) > L):
        raise ValueError("every length must lie in (%d, %d]" % (lo, L))
    full = np.broadcast_to(arr.reshape(arr.shape + (1,) * (len(lead) - arr.ndim)), lead)
    return np.ascontiguousarray(full, dtype=np.int32).reshape(-1)


def _lengths_args(host, device):
    """(device int32 tensor, ctypes pointer to the host copy) of host lengths."""
    host = np.require(host, dtype=np.int32, requirements=("C", "W"))
    return (torch.from_numpy(host).to(device), host.ctypes.data_as(_lib.c_int_p))


@_on_device
def stft_lengths(x, lengths, n_fft=512):
    """x [..., L] float32, signals of their own lengths (zero after) -> Y [..., T, F] complex64, T = 1 + L // hop.
    lengths: per signal, or per leading index repeated over the remaining axes (see signal_lengths); every length in
    (n_fft / 2, L].  Frame t < 1 + length // hop of a signal is stft() of the signal trimmed to its length (reflect
    padding at its own end); later frames are 0."""
    _need(x, torch.float32, "x")
    L = x.shape[-1]
    n_sig = x.numel() // L
    host = signal_lengths(lengths, x.shape[:-1], L, lo=n_fft // 2)
    T, F = n_frames(L, n_fft), n_fft // 2 + 1
    Y = torch.empty(x.shape[:-1] + (T, F), dtype=torch.complex64, device=x.device)
    dev, hp = _lengths_args(host, x.device)
    _lib.check(_lib.load().disco_stft_lengths(_ptr(x), _ptr(dev), hp, _ptr(Y), n_sig, L, n_fft, _stream()))
    return Y


@_on_device
def istft_lengths(Y, lengths, length, n_fft=512):
    """Y [..., T, F] complex64 -> x [..., length] float32, each signal of its own length: samples < lengths[s] are
    istft(Y_s[:1 + lengths[s] // hop], lengths[s]), the rest 0.  lengths as in stft_lengths, each in (0, length]."""
    _need(Y, torch.complex64, "Y")
    T, F = Y.shape[-2:]
    if F != n_fft // 2 + 1:
        raise ValueError("last dimension must be n_fft/2 + 1 bins")
    n_sig = Y.numel() // (T * F)
    host = signal_lengths(lengths, Y.shape[:-2], int(length))
    x = torch.empty(Y.shape[:-2] + (int(length),), dtype=torch.float32, device=Y.device)
    dev, hp = _lengths_args(host, Y.device)
    _lib.check(_lib.load().disco_istft_lengths(_ptr(Y), _ptr(dev), hp, _ptr(x), n_sig, T, int(length), n_fft,
                                               _stream()))
    return x


@_on_device
def scm_recursive(Y, mask, Z=None, lambda_cor=0.95, block=8, power=2, R0=None, n_fft=512, node_sel=None,
                  frames=None):
    """Exponentially smoothed SCM pair, R <- lambda R + (1 - lambda) w x x^H per frame (reference
    spatial_correlation_matrix, internal_formulas.py:84-103), sampled after every block of `block` frames.
    Y [B, Ksel, C, T, F], Z [B, K, T, F] or None, mask [B, Ksel, T, F] or None, R0 = (R0ss, R0nn) [B, Ksel, F, D, D]
    -> Rss, Rnn [B, Ksel, J, F, D, D], J = ceil(T / block), D = C + K - 1 <= 16.  At D >= 9 only the upper triangle
    and the real diagonal of R0 are read (R0 is Hermitian); the values are those of the D <= 8 two-level scan.
    frames: None, or host integers, one per utterance in [1, T]: utterance b then has frames[b] frames, its blocks
    j < ceil(frames[b] / block) equal the call on Y[b, ..., :frames[b], :] alone bit for bit, its later blocks are 0,
    and no frame from frames[b] on is read."""
    n_utt, K, sel, n_sel, _ = _cat_args(Y, Z, node_sel, n_fft)
    if mask is not None:
        _need(mask, torch.float32, "mask")
    B, Ks, C, T, F = Y.shape
    D = C + K - 1
    if mask is not None and tuple(mask.shape) != (B, Ks, T, F):
        raise ValueError("mask shape %s, expected %s" % (tuple(mask.shape), (B, Ks, T, F)))
    J = (T + block - 1) // block
    Rss = torch.empty((B, Ks, J, F, D, D), dtype=torch.complex64, device=Y.device)
    Rnn = torch.empty_like(Rss)
    r0s = r0n = None
    if R0 is not None:
        r0s, r0n = R0
        for r in (r0s, r0n):
            _need(r, torch.complex64, "R0")
            if tuple(r.shape) != (B, Ks, F, D, D):
                raise ValueError("R0 shape %s, expected %s" % (tuple(r.shape), (B, Ks, F, D, D)))
    if frames is None:
        _lib.check(_lib.load().disco_scm_recursive(_ptr(Y), _ptr(Z), _ptr(mask), _ptr(r0s), _ptr(r0n), _ptr(Rss),
                                                   _ptr(Rnn), float(lambda_cor), int(block), int(power), n_utt, K, C,
                                                   T, n_fft, sel, n_sel, _stream()))
    else:
        dev, hp = _lengths_args(signal_lengths(frames, (B, n_utt // B), T), Y.device)   # n_utt = B * Ksel if Z is None
        _lib.check(_lib.load().disco_scm_recursive_lengths(_ptr(Y), _ptr(Z), _ptr(mask), _ptr(r0s), _ptr(r0n),
                                                           _ptr(Rss), _ptr(Rnn), float(lambda_cor), int(block),
                                                           int(power), n_utt, K, C, T, n_fft, sel, n_sel, _ptr(dev),
                                                           hp, _stream()))
    return Rss, Rnn


@_on_device
def filter_sum_blocks(W, Y, Z=None, block=8, lag=1, conj=True, ref=0, n_fft=512, node_sel=None, frames=None):
    """One filter per block of frames: out[t] = W[t // block - lag]^H x[t] (pass-through of channel `ref` while no
    filter exists yet).  W [B, Ksel, J, F, D], D = C + K - 1 <= 16 -> out, resid = x[ref] - out, [B, Ksel, T, F].
    frames: None, or host integers, one per utterance in [1, T]: frames t < frames[b] of utterance b are the call on
    its first frames[b] frames alone (reading only W[b, :, :ceil(frames[b] / block)]); later frames are 0."""
    _need(W, torch.complex64, "W")
    n_utt, K, sel, n_sel, _ = _cat_args(Y, Z, node_sel, n_fft)
    B, Ks, C, T, F = Y.shape
    D, J = C + K - 1, (T + block - 1) // block
    if tuple(W.shape) != (B, Ks, J, F, D):
        raise ValueError("W shape %s, expected %s" % (tuple(W.shape), (B, Ks, J, F, D)))
    out = torch.empty((B, Ks, T, F), dtype=torch.complex64, device=Y.device)
    resid = torch.empty_like(out)
    if frames is None:
        _lib.check(_lib.load().disco_filter_sum_blocks(_ptr(W), 1 if conj else 0, _ptr(Y), _ptr(Z), _ptr(out),
                                                       _ptr(resid), int(ref), int(block), int(lag), n_utt, K, C, T,
                                                       n_fft, sel, n_sel, _stream()))
    else:
        dev, hp = _lengths_args(signal_lengths(frames, (B, n_utt // B), T), Y.device)   # n_utt = B * Ksel if Z is None
        _lib.check(_lib.load().disco_filter_sum_blocks_lengths(_ptr(W), 1 if conj else 0, _ptr(Y), _ptr(Z), _ptr(out),
                                                               _ptr(resid), int(ref), int(block), int(lag), n_utt, K,
                                                               C, T, n_fft, sel, n_sel, _ptr(dev), hp, _stream()))
    return out, resid


@_on_device
def stream_stft(hist, chunk, length, t0, n_fr, n_fft=512, hist_out=None, Y_blk=None, blk_slot=0, final=False):
    """Frames [t0, t0 + n_fr) of signals that arrive chunk by chunk, equal to those of stft() on the whole signal.
    hist [..., n_fft] float32 holds samples [L0 - n_fft, L0) of every signal, chunk [..., n] the new samples
    [L0, length) (n = 0 on the final call, final=True, which reflects the last frame at the end).  hist_out [...,
    n_fft] (optional) receives samples [length - n_fft, length); Y_blk [..., P, F] (optional) receives the frames at
    slots blk_slot ...  Returns Y [..., n_fr, F] complex64."""
    _need(hist, torch.float32, "hist")
    _need(chunk, torch.float32, "chunk")
    lead, F = tuple(hist.shape[:-1]), n_fft // 2 + 1
    if hist.shape[-1] != n_fft or tuple(chunk.shape[:-1]) != lead:
        raise ValueError("hist %s / chunk %s, expected [..., %d] / [..., n] with the same leading shape"
                         % (tuple(hist.shape), tuple(chunk.shape), n_fft))
    n_sig = hist.numel() // n_fft
    P = 0
    if hist_out is not None:
        _need(hist_out, torch.float32, "hist_out")
        if hist_out.shape != hist.shape or hist_out.data_ptr() == hist.data_ptr():
            raise ValueError("hist_out must be a second buffer shaped like hist")
    if Y_blk is not None:
        _need(Y_blk, torch.complex64, "Y_blk")
        P = Y_blk.shape[-2]
        if tuple(Y_blk.shape) != lead + (P, F):
            raise ValueError("Y_blk shape %s, expected %s" % (tuple(Y_blk.shape), lead + (P, F)))
    n_sig, n_new, P = _c_int(n_sig, "n_sig"), _c_int(chunk.shape[-1], "chunk length"), _c_int(P, "Y_blk frames")
    r = _records(_scalar_record((length, n_new, t0, n_fr, blk_slot, 1 if final else 0, 0, 0)), 1, STFT_SLOT_FIELDS,
                 "record", n_fft)[0]
    Y = torch.empty(lead + (int(n_fr), F), dtype=torch.complex64, device=hist.device)
    _lib.check(_lib.load().disco_stream_stft(_ptr(hist), _ptr(chunk) if chunk.numel() else None, _ptr(hist_out),
                                             _ptr(Y), _ptr(Y_blk), n_sig, n_new, int(r[0]), int(r[2]), int(r[3]), P,
                                             int(r[4]), int(r[5]), n_fft, _stream()))
    return Y


@_on_device
def stream_istft(Y, carry, t0, length, n_fft=512, final=False, x=None, x_first=0):
    """The hop blocks that frames [t0, t0 + n_fr) of Y [..., n_fr, F] make final, equal to those of istft() on the
    whole signal: samples [(max(t0, 1) - 1) hop, (t0 + n_fr - 1) hop), and with final=True the rest up to `length`.
    carry [..., n_fft // 2] float32 (zeros before frame 0) is updated in place.  They are written to x [..., S] at
    x[..., s - x_first] (x = None: a new tensor starting at the first sample written).  Returns x."""
    _need(Y, torch.complex64, "Y")
    _need(carry, torch.float32, "carry")
    n_fr, F = Y.shape[-2:]
    H = n_fft // 2
    lead = tuple(Y.shape[:-2])
    if F != H + 1 or tuple(carry.shape) != lead + (H,):
        raise ValueError("Y %s / carry %s, expected [..., n_fr, %d] / [..., %d]" % (tuple(Y.shape), tuple(carry.shape),
                                                                                    H + 1, H))
    n_sig = carry.numel() // H
    lo = max(int(t0) - 1, 0) * H
    hi = min(int(length), int(length) if final else (int(t0) + n_fr - 1) * H)
    if x is None:
        x_first = lo
    else:
        _need(x, torch.float32, "x")
        if tuple(x.shape[:-1]) != lead:
            raise ValueError("x shape %s, expected %s" % (tuple(x.shape), lead + (-1,)))
    n_sig = _c_int(n_sig, "n_sig")
    s_max = _c_int(max(hi - lo, 0) if x is None else x.shape[-1], "x length")
    r = _records(_scalar_record((t0, n_fr, length, 1 if final else 0, x_first)), 1, ISTFT_SLOT_FIELDS, "record",
                 n_fft)[0]
    if x is None:
        x = torch.empty(lead + (s_max,), dtype=torch.float32, device=Y.device)
    _lib.check(_lib.load().disco_stream_istft(_ptr(Y) if Y.numel() else None, _ptr(carry), _ptr(x) if x.numel() else None,
                                              n_sig, int(r[0]), int(r[1]), int(r[2]), int(r[3]), int(r[4]), s_max,
                                              n_fft, _stream()))
    return x


STFT_SLOT_FIELDS = ("length", "n_new", "t0", "n_fr", "blk_slot", "final", "hist_sel", "hist_write")
ISTFT_SLOT_FIELDS = ("t0", "n_fr", "length", "final", "x_first")
INT_MAX = 2 ** 31 - 1


def max_stream_length(n_fft=512):
    """The largest sample position of a stream record the library accepts, relative to the record's origin, and the
    longest whole signal its STFT / iSTFT take: the kernels form positions up to a frame and a CTA stride past it in
    C int.  The stream ops rebase their records (_rebase), so a stream itself may run without an end."""
    return INT_MAX - n_fft - 1024


def _c_int(v, name):
    v = int(v)
    if not -INT_MAX - 1 <= v <= INT_MAX:
        raise ValueError("%s = %d does not fit in a C int" % (name, v))
    return v


def _scalar_record(values):
    """One record [1, n] of host integers of any size (ValueError past int64)."""
    try:
        return np.array([[int(v) for v in values]], dtype=np.int64)
    except OverflowError:
        raise ValueError("a stream position does not fit in 64 bits: %s" % (values,)) from None


def _rebase(rec, fields, n_fft):
    """Absolute stream records [n_slot, len(fields)] (int64) relative to an origin O per slot.

    O is a multiple of the hop H; it lies at or before every sample the call reads, writes or carries: the history
    start length - n_new - n_fft and the first sample (t0 - 1) H of frame t0 (STFT); the first sample (t0 - 1) H of
    hop block t0, x_first and length - 1 (iSTFT).  O = 0 whenever the call can reach the start reflection (t0 = 0, or
    fewer than n_fft samples before the chunk).  length and x_first lose O, t0 loses O / H.  The kernels use positions
    only to address the history, the chunk and x and to place the two reflections, so a call's outputs do not depend
    on O, and a valid record stays valid.  Formed without a product, so no int64 position overflows."""
    H = n_fft // 2
    rec = rec.copy()
    if H < 1:                 # no such transform: the library rejects the call
        return rec
    if fields is STFT_SLOT_FIELDS:
        length, n_new, t0 = rec[:, 0], rec[:, 1], rec[:, 2]
        o = np.maximum(np.minimum((length - n_new - n_fft) // H, t0 - 1), 0)
        rec[:, 0] -= o * H
        rec[:, 2] -= o
    else:
        t0, length, x_first = rec[:, 0], rec[:, 2], rec[:, 4]
        o = np.maximum(np.minimum(np.minimum(t0 - 1, x_first // H), (length - 1) // H), 0)
        rec[:, 0] -= o
        rec[:, 2] -= o * H
        rec[:, 4] -= o * H
    return rec


def _records(slots, n_slot, fields, name, n_fft):
    """Per-slot records [n_slot, len(fields)] of absolute positions, rebased (_rebase), as a contiguous host int32
    array.  ValueError for a field that does not fit in a C int after rebasing: nothing is narrowed silently."""
    arr = np.asarray(slots)
    if arr.dtype.kind == "O" and arr.size and all(isinstance(v, int) for v in arr.ravel()):
        raise ValueError("%s: a position does not fit in 64 bits" % name)
    if arr.dtype.kind not in "iu":
        raise TypeError("%s must be integers, got %s" % (name, arr.dtype))
    if tuple(arr.shape) != (n_slot, len(fields)):
        raise ValueError("%s shape %s, expected (%d, %d): %s" % (name, tuple(arr.shape), n_slot, len(fields),
                                                                ", ".join(fields)))
    if arr.dtype.kind == "u" and arr.size and arr.max() > np.iinfo(np.int64).max:
        raise ValueError("%s: a position does not fit in 64 bits" % name)
    rec = _rebase(arr.astype(np.int64), fields, n_fft)
    bad = (rec < -INT_MAX - 1) | (rec > INT_MAX)
    if bad.any():
        s, f = np.argwhere(bad)[0]
        raise ValueError("%s: slot %d's %s = %d does not fit in a C int, even relative to the stream's origin"
                         % (name, s, fields[f], rec[s, f]))
    return np.ascontiguousarray(rec, dtype=np.int32)


@_on_device
def stream_stft_slots(hist, chunk, slots, f_max, n_fft=512, Y_blk=None):
    """stream_stft on a pool of independent streams, one record per slot (STFT_SLOT_FIELDS): slot s holds the signals
    chunk[s] ([S, ..., n_max] float32, its new samples at the start of each row).  hist [2, S, ..., n_fft] float32 holds
    two history buffers: slot s reads buffer hist_sel and, with hist_write, writes its new history to the other one.
    Y_blk [S, ..., P, F] (optional) receives the frames at rows blk_slot ...  Returns Y [S, ..., f_max, F]: frames t0
    .. t0 + n_fr - 1 of slot s at rows 0 .. n_fr - 1 (later rows are not written).  Signals are paired inside a slot,
    so each slot equals stream_stft on that slot alone."""
    _need(hist, torch.float32, "hist")
    _need(chunk, torch.float32, "chunk")
    lead, F = tuple(chunk.shape[:-1]), n_fft // 2 + 1
    if len(lead) < 1 or tuple(hist.shape) != (2,) + lead + (n_fft,):
        raise ValueError("hist %s / chunk %s, expected [2, S, ..., %d] / [S, ..., n_max]"
                         % (tuple(hist.shape), tuple(chunk.shape), n_fft))
    S = lead[0]
    n_sig = int(np.prod(lead[1:], dtype=np.int64))
    P = 0
    if Y_blk is not None:
        _need(Y_blk, torch.complex64, "Y_blk")
        P = Y_blk.shape[-2]
        if tuple(Y_blk.shape) != lead + (P, F):
            raise ValueError("Y_blk shape %s, expected %s" % (tuple(Y_blk.shape), lead + (P, F)))
    host = _records(slots, S, STFT_SLOT_FIELDS, "slots", n_fft)
    n_sig, n_max = _c_int(n_sig, "n_sig"), _c_int(chunk.shape[-1], "chunk length")
    f_max, P = _c_int(f_max, "f_max"), _c_int(P, "Y_blk frames")
    Y = torch.empty(lead + (f_max, F), dtype=torch.complex64, device=hist.device)
    dev = torch.from_numpy(host).to(hist.device)
    _lib.check(_lib.load().disco_stream_stft_slots(_ptr(hist), _ptr(chunk) if chunk.numel() else None,
                                                   _ptr(Y) if Y.numel() else None, _ptr(Y_blk), _ptr(dev),
                                                   host.ctypes.data_as(_lib.c_int_p), S, n_sig, n_max, f_max, P, n_fft,
                                                   _stream()))
    return Y


@_on_device
def stream_istft_slots(Y, carry, slots, x, n_fft=512):
    """stream_istft on a pool of independent streams, one record per slot (ISTFT_SLOT_FIELDS): frames t0 .. t0 + n_fr -
    1 of slot s are Y[s] [S, ..., f_max, F] rows 0 .. n_fr - 1; carry [S, ..., n_fft // 2] is updated in place; the
    samples that become final are written to x [S, ..., s_max] at x[s, ..., i - x_first].  A slot with n_fr = 0 that
    is not final is left as it is.  Each slot equals stream_istft on that slot alone.  Returns x."""
    _need(Y, torch.complex64, "Y")
    _need(carry, torch.float32, "carry")
    _need(x, torch.float32, "x")
    f_max, F = Y.shape[-2:]
    H = n_fft // 2
    lead = tuple(Y.shape[:-2])
    if F != H + 1 or len(lead) < 1 or tuple(carry.shape) != lead + (H,) or tuple(x.shape[:-1]) != lead:
        raise ValueError("Y %s / carry %s / x %s, expected [S, ..., f_max, %d] / [S, ..., %d] / [S, ..., s_max]"
                         % (tuple(Y.shape), tuple(carry.shape), tuple(x.shape), H + 1, H))
    S = lead[0]
    n_sig = int(np.prod(lead[1:], dtype=np.int64))
    host = _records(slots, S, ISTFT_SLOT_FIELDS, "slots", n_fft)
    n_sig, f_max, s_max = _c_int(n_sig, "n_sig"), _c_int(f_max, "f_max"), _c_int(x.shape[-1], "x length")
    dev = torch.from_numpy(host).to(Y.device)
    _lib.check(_lib.load().disco_stream_istft_slots(_ptr(Y) if Y.numel() else None, _ptr(carry),
                                                    _ptr(x) if x.numel() else None, _ptr(dev),
                                                    host.ctypes.data_as(_lib.c_int_p), S, n_sig, f_max, s_max, n_fft,
                                                    _stream()))
    return x


@_on_device
def band_stats(x, ba, sel=None):
    """IIR filter bank + statistics of every band's output (reference metrics.py:96-110: lfilter, then np.var of
    the selected samples).  x [..., L] float32 (a time slice of a contiguous tensor is taken in place),
    ba [n_band, 2, order+1] float64 (b, a), sel optional like x -> stats [..., n_band, 3] float64: count, sum,
    sum of squares of the selected filter outputs."""
    for t, name in ((x, "x"), (sel, "sel")):
        if t is None:
            continue
        if not isinstance(t, torch.Tensor) or not t.is_cuda:
            raise TypeError("%s must be a CUDA tensor (disco_b200 has no CPU path)" % name)
        if t.dtype != torch.float32:
            raise TypeError("%s must be float32" % name)
    L, lead = x.shape[-1], tuple(x.shape[:-1])
    xv = x.reshape(-1, L)                      # a view when the rows are equally spaced
    if xv.stride(1) != 1 or (xv.shape[0] > 1 and xv.stride(0) < L):
        xv = xv.contiguous()
    ld = xv.stride(0) if xv.shape[0] > 1 else L
    sv = None
    if sel is not None:
        if tuple(sel.shape) != tuple(x.shape):
            raise ValueError("sel must have the shape of x")
        sv = torch.empty_strided(xv.shape, (ld, 1), dtype=torch.float32, device=x.device)
        sv.copy_(sel.reshape(-1, L))
    if not isinstance(ba, torch.Tensor) or ba.is_complex():
        raise TypeError("ba must be a real tensor [n_band, 2, order + 1]")
    ba = ba.to(device=x.device, dtype=torch.float64).contiguous()
    if ba.dim() != 3 or ba.shape[1] != 2:
        raise ValueError("ba must be [n_band, 2, order + 1]")
    n_band, order = ba.shape[0], ba.shape[2] - 1
    stats = torch.empty(lead + (n_band, 3), dtype=torch.float64, device=x.device)
    _lib.check(_lib.load().disco_band_stats(_ptr(xv), _ptr(sv) if sv is not None else None, _ptr(ba), _ptr(stats),
                                            xv.shape[0], L, int(ld), n_band, order, _stream()))
    return stats


# Device scratch of one disco_bss_eval call (the Gram matrices and their factors, ~11 MB per reference set of 2
# sources at flen 512); larger batches of sets run in consecutive chunks.
BSS_WORKSPACE_CAP = 1 << 30


@_on_device
def bss_eval(refs, ests, flen=512):
    """Float64 projection norms of BSS-eval (disco_bss_eval).  refs [S, nsrc, L], ests [S, R, L] float32 (R estimate
    rows per reference set) -> norms [S, R, 1 + 2 nsrc] float64: ‖e‖², the part of ‖P_all e‖² from each reference's
    block, ‖P_k e‖² of each reference alone.  Sets are processed in chunks whose workspace stays within
    BSS_WORKSPACE_CAP bytes (one set at least)."""
    _need(refs, torch.float32, "refs")
    _need(ests, torch.float32, "ests")
    if refs.dim() != 3 or ests.dim() != 3 or ests.shape[0] != refs.shape[0] or ests.shape[2] != refs.shape[2]:
        raise ValueError("refs [S, nsrc, L] / ests [S, R, L] shape mismatch: %s / %s"
                         % (tuple(refs.shape), tuple(ests.shape)))
    S, nsrc, L = refs.shape
    R = ests.shape[1]
    if nsrc > 4:
        raise NotImplementedError("bss_eval: at most 4 reference sources (got %d)" % nsrc)
    lib = _lib.load()
    norms = torch.empty((S, R, 1 + 2 * nsrc), dtype=torch.float64, device=refs.device)
    if S == 0:
        return norms
    per_set = lib.disco_bss_eval_workspace(1, nsrc, R, L, int(flen))
    if per_set == 0:
        _lib.check(lib.disco_bss_eval(None, None, None, 1, nsrc, R, L, int(flen), None, 0, _stream()))
    chunk = max(1, min(S, BSS_WORKSPACE_CAP // per_set))
    ws_bytes = lib.disco_bss_eval_workspace(chunk, nsrc, R, L, int(flen))
    ws = torch.empty(ws_bytes // 8, dtype=torch.float64, device=refs.device)
    for s0 in range(0, S, chunk):
        n = min(chunk, S - s0)
        _lib.check(lib.disco_bss_eval(_ptr(refs[s0:s0 + n]), _ptr(ests[s0:s0 + n]), _ptr(norms[s0:s0 + n]), n, nsrc,
                                      R, L, int(flen), _ptr(ws), ws_bytes, _stream()))
    return norms


@_on_device
def resample_poly(x, taps, up, down, lengths=None):
    """scipy.signal.resample_poly(x, up, down, window=taps) along the last axis (disco_resample_poly).
    x [..., L] float32, taps [n] float64 (scipy's `window`; the gain `up` is applied inside) -> [..., ceil(L up / down)]
    float64.  up and down are reduced by their gcd first, as scipy does; equal rates return x as float64.
    lengths (per signal, or per leading index as in signal_lengths; each in (0, L]): row s is its first lengths[s]
    samples, and its output is resample_poly of that trimmed row followed by zeros (disco_resample_poly_lengths)."""
    _need(x, torch.float32, "x")
    _need(taps, torch.float64, "taps")
    up, down = int(up), int(down)
    if up < 1 or down < 1:
        raise ValueError("up and down must be >= 1")
    g = math.gcd(up, down)
    up, down = up // g, down // g
    L = x.shape[-1]
    host = None if lengths is None else signal_lengths(lengths, x.shape[:-1], L)
    if up == down == 1:
        return x.double()    # rows are zero after their lengths already
    n_out = -(-L * up // down)
    y = torch.empty(x.shape[:-1] + (n_out,), dtype=torch.float64, device=x.device)
    n_sig = x.numel() // L if L else 0
    if n_sig == 0:
        return y
    if host is None:
        _lib.check(_lib.load().disco_resample_poly(_ptr(x), _ptr(y), _ptr(taps), taps.numel(), up, down, n_sig, L,
                                                   _stream()))
    else:
        dev, hp = _lengths_args(host, x.device)
        _lib.check(_lib.load().disco_resample_poly_lengths(_ptr(x), _ptr(y), _ptr(taps), taps.numel(), up, down, n_sig,
                                                           L, _ptr(dev), hp, _stream()))
    return y


# Device scratch of one disco_stoi call (energies and kept-frame lists of every clean, band envelopes of every clean
# and every pair: ~85 KB per spectrogram of 9 s); larger batches of pairs run in consecutive chunks.
STOI_WORKSPACE_CAP = 1 << 30


@_on_device
def stoi(cleans, degraded, pairs, lengths=None):
    """Classic STOI of 10 kHz signals (disco_stoi).  cleans [C, L], degraded [D, L] float64, pairs [P, 2] int32
    (clean index, degraded index) -> d [P] float64 (1e-5 below 30 STFT frames), n_sel [C] int32 (frames kept by the
    silent-frame removal; -1 for a clean no pair names), n_frames [P] int32 (STFT frames scored).  Pairs are processed
    in chunks whose workspace stays within STOI_WORKSPACE_CAP bytes (one pair at least); a chunk computes only the
    cleans its pairs name, each once.  lengths [C] (each in [256, L], or None): clean c and every degraded signal
    paired with it are their first lengths[c] samples (disco_stoi_lengths); None scores whole rows."""
    _need(cleans, torch.float64, "cleans")
    _need(degraded, torch.float64, "degraded")
    _need(pairs, torch.int32, "pairs")
    if cleans.dim() != 2 or degraded.dim() != 2 or pairs.dim() != 2 or pairs.shape[1] != 2 or \
            degraded.shape[1] != cleans.shape[1]:
        raise ValueError("cleans [C, L] / degraded [D, L] / pairs [P, 2] shape mismatch: %s / %s / %s"
                         % (tuple(cleans.shape), tuple(degraded.shape), tuple(pairs.shape)))
    C, L = cleans.shape
    D, P = degraded.shape[0], pairs.shape[0]
    if L < 256:
        raise ValueError("stoi: signals of %d samples at 10 kHz; at least 256 are needed" % L)
    dev = cleans.device
    d = torch.empty(P, dtype=torch.float64, device=dev)
    n_frames = torch.empty(P, dtype=torch.int32, device=dev)
    n_sel = torch.full((C,), -1, dtype=torch.int32, device=dev)
    if P == 0:
        return d, n_sel, n_frames
    if C == 0 or D == 0 or int(pairs[:, 0].min()) < 0 or int(pairs[:, 0].max()) >= C or \
            int(pairs[:, 1].min()) < 0 or int(pairs[:, 1].max()) >= D:
        raise IndexError("stoi: pair indices out of range (%d cleans, %d degraded signals)" % (C, D))
    lib = _lib.load()
    host = None if lengths is None else signal_lengths(lengths, (C,), L, lo=255)

    def run(cl, pr, d_out, sel_out, nf_out, n_cl, n_pr, ws, ws_bytes, hl):
        if hl is None:
            _lib.check(lib.disco_stoi(_ptr(cl), _ptr(degraded), _ptr(pr), _ptr(d_out), _ptr(sel_out), _ptr(nf_out),
                                      n_cl, D, n_pr, L, _ptr(ws), ws_bytes, _stream()))
        else:
            ld, hp = _lengths_args(hl, dev)
            _lib.check(lib.disco_stoi_lengths(_ptr(cl), _ptr(degraded), _ptr(pr), _ptr(d_out), _ptr(sel_out),
                                              _ptr(nf_out), n_cl, D, n_pr, L, _ptr(ld), hp, _ptr(ws), ws_bytes,
                                              _stream()))

    per_pair = lib.disco_stoi_workspace(1, 1, L)
    if per_pair == 0:
        _lib.check(lib.disco_stoi(None, None, None, None, None, None, 1, 1, 1, L, None, 0, _stream()))
    if lib.disco_stoi_workspace(C, P, L) <= STOI_WORKSPACE_CAP:
        ws_bytes = lib.disco_stoi_workspace(C, P, L)
        ws = torch.empty(ws_bytes // 8 + 1, dtype=torch.float64, device=dev)
        run(cleans, pairs, d, n_sel, n_frames, C, P, ws, ws_bytes, host)
        named = torch.zeros(C, dtype=torch.bool, device=dev)
        named[pairs[:, 0].long()] = True
        return d, n_sel.masked_fill_(~named, -1), n_frames
    chunk = max(1, STOI_WORKSPACE_CAP // per_pair)
    ws_bytes = lib.disco_stoi_workspace(min(chunk, C), chunk, L)
    ws = torch.empty(ws_bytes // 8 + 1, dtype=torch.float64, device=dev)
    for p0 in range(0, P, chunk):
        n = min(chunk, P - p0)
        used, local = torch.unique(pairs[p0:p0 + n, 0], return_inverse=True)
        sub = cleans.index_select(0, used)
        pr = torch.stack((local.to(torch.int32), pairs[p0:p0 + n, 1]), dim=1).contiguous()
        sel = torch.empty(used.numel(), dtype=torch.int32, device=dev)
        hl = None if host is None else np.ascontiguousarray(host[used.cpu().numpy()])
        run(sub, pr, d[p0:], sel, n_frames[p0:], used.numel(), n, ws, ws_bytes, hl)
        n_sel[used] = sel
    return d, n_sel, n_frames


@_on_device
def transpose_last2(a):
    """[..., R, C] -> [..., C, R] (contiguous) for complex64 / float32 device tensors."""
    R, Cc = a.shape[-2:]
    batch = a.numel() // (R * Cc) if a.numel() else 0
    out = torch.empty(a.shape[:-2] + (Cc, R), dtype=a.dtype, device=a.device)
    lib = _lib.load()
    if a.dtype == torch.complex64:
        _need(a, torch.complex64, "a")
        _lib.check(lib.disco_transpose_c64(_ptr(a), _ptr(out), batch, R, Cc, _stream()))
    else:
        _need(a, torch.float32, "a")
        _lib.check(lib.disco_transpose_f32(_ptr(a), _ptr(out), batch, R, Cc, _stream()))
    return out


@_on_device
def apply_mask(X, m, one_minus=False):
    """m * X or (1 - m) * X, complex64 x float32.  Same shapes, or X [..., C, T, F] with one mask plane
    m [..., T, F] shared by the C channels of a group (one launch either way)."""
    _need(X, torch.complex64, "X")
    _need(m, torch.float32, "m")
    out = torch.empty_like(X)
    lib = _lib.load()
    if X.shape == m.shape:
        _lib.check(lib.disco_apply_mask(_ptr(X), _ptr(m), _ptr(out), X.numel(), 1 if one_minus else 0, _stream()))
    elif X.dim() == m.dim() + 1 and tuple(X.shape[:-3]) + tuple(X.shape[-2:]) == tuple(m.shape):
        plane = X.shape[-1] * X.shape[-2]
        _lib.check(lib.disco_apply_mask_channels(_ptr(X), _ptr(m), _ptr(out), m.numel() // plane, X.shape[-3], plane,
                                                 1 if one_minus else 0, _stream()))
    else:
        raise ValueError("shape mismatch")
    return out
