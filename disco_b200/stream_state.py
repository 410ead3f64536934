"""The saved state of live online Tango sessions: one format for OnlineTangoStream and OnlineTangoPool.

A session state is a plain nested dict of tensors, ints, floats, strings, tuples, lists, dicts and None, so that
torch.save / torch.load(weights_only=True) round-trip it.  It holds B >= 1 lockstep streams (a pool slot: B = 1):

    version, kind            VERSION; "clean" for a stream with clean components, "plain" otherwise
    n_fft, lambda_cor, block, lag, mu, rank, ref_mic, filter_type, mask_for_z, clean, vads, wide
                             the options (wide: D > 8, the stacks that take the staged scan)
    K, C, channels           the geometry: C an int and channels None, or C None and channels K per-node counts
    B                        the number of streams
    samples_in, frames_out, samples_out, closed
                             Python ints: (frames_out, samples_out) = emission(samples_in), closed = frames_out // block
    groups                   per channel-count group (ascending counts, as ragged._Layout orders them), a dict:
        C, nodes             the count and the group's nodes
        hist                 [B, n, C, n_fft] float32: samples [samples_in - n_fft, samples_in), 0 before sample 0
        hist_s, hist_n       the same for the clean components (None without them)
        Yblk                 [B, n, C, block, F] complex64: the open block's spectra (frames closed * block on)
        Sblk, Nblk           those of s and n under 'use_oracle_*' (None otherwise)
        R1, R2               [R_ss, R_nn] [B, n, F, C, C] / [B, n, F, D, D] complex64 after the last closed block, or
                             None while closed = 0 and no R0 seeds them (the scan starts from 0)
        W1, W2               [B, nw, n, F, C] / [B, nw, n, F, D] complex64: the filters of blocks closed - nw ..
                             closed - 1, nw = min(closed, lag): those a later block still reads (block j reads
                             W_(j - lag); before block 0's filter exists, the kernel's pass-through)
    m1, m2                   [B, K, block, F] float32: the open block's masks over all K nodes
    zblk                     [B, K, block, F] complex64: its step-1 output (None for K = 1)
    zsblk, znblk             its z_s, z_n ('compressed' / 'use_oracle_zs' with K > 1; None otherwise)
    carry                    [B, 6 or 1, K, n_fft / 2] float32: the iSTFT carry of each time signal (TIME_NAMES with
                             clean components, yf alone otherwise)

The format does not depend on the class that wrote it.  Entries of the block buffers past the open block's frames are
stale (never read before they are written); they are kept as they are.  check() validates a state on the host and
raises ValueError naming the offending field; concat() joins states of identical options, geometry and counters into
one state of B = sum(B_i) streams."""
import numbers

import torch

VERSION = 1
OPTIONS = ("n_fft", "lambda_cor", "block", "lag", "mu", "rank", "ref_mic", "filter_type", "mask_for_z", "clean",
           "vads", "wide")
GEOMETRY = ("K", "C", "channels")
COUNTERS = ("samples_in", "frames_out", "samples_out", "closed")
KEYS = ("version", "kind") + OPTIONS + GEOMETRY + ("B",) + COUNTERS + \
    ("groups", "m1", "m2", "zblk", "zsblk", "znblk", "carry")
GROUP_KEYS = ("C", "nodes", "hist", "hist_s", "hist_n", "Yblk", "Sblk", "Nblk", "R1", "R2", "W1", "W2")
N_TIME = 6                      # len(stream.TIME_NAMES)


def _fail(field, what):
    raise ValueError("session state: %s %s" % (field, what))


def _int(state, field, low=0):
    v = state[field]
    if isinstance(v, bool) or not isinstance(v, numbers.Integral) or v < low:
        _fail(field, "must be an integer >= %d, got %r" % (low, v))
    return int(v)


def _tensor(x, field, shape, dtype):
    if not isinstance(x, torch.Tensor):
        _fail(field, "must be a tensor, got %s" % type(x).__name__)
    if x.dtype != dtype or tuple(x.shape) != tuple(shape):
        _fail(field, "must be %s [%s], got %s [%s]" % (str(dtype).replace("torch.", ""), ", ".join(map(str, shape)),
                                                        str(x.dtype).replace("torch.", ""),
                                                        ", ".join(map(str, x.shape))))


def _optional(x, field, shape, dtype, present):
    """A tensor that exists exactly when `present`."""
    if not present:
        if x is not None:
            _fail(field, "must be None for these options")
    else:
        _tensor(x, field, shape, dtype)


def _pair(x, field, shape, allow_none):
    """[R_ss, R_nn] complex64 tensors of `shape`, or None where allowed."""
    if x is None:
        if not allow_none:
            _fail(field, "must hold the carried matrices once a block has closed")
        return
    if not isinstance(x, (tuple, list)) or len(x) != 2:
        _fail(field, "must be the pair [R_ss, R_nn] or None")
    for i, r in enumerate(x):
        _tensor(r, "%s[%d]" % (field, i), shape, torch.complex64)


def _layout(state):
    """ragged._Layout of the state's geometry (ValueError for a bad one)."""
    from .ragged import _Layout
    K = _int(state, "K", 1)
    C, channels = state["C"], state["channels"]
    if (C is None) == (channels is None):
        _fail("C", "or channels: exactly one of them is given")
    if channels is None:
        C = _int(state, "C", 1)
        counts = [C] * K
    else:
        if not isinstance(channels, list):
            _fail("channels", "must be a list of K counts")
        counts = channels
    try:
        lay = _Layout(counts, None, state["ref_mic"])
    except (TypeError, NotImplementedError, ValueError) as e:
        _fail("channels" if channels is not None else "C", "/ ref_mic: %s" % e)
    if lay.K != K:
        _fail("channels", "holds %d counts for K = %d" % (lay.K, K))
    return lay


def _check_options(state):
    from .stream import _check_options as check_opts, _check_params
    for f in ("n_fft", "block", "lag", "ref_mic"):
        _int(state, f, 0)
    for f in ("lambda_cor", "mu"):
        if isinstance(state[f], bool) or not isinstance(state[f], numbers.Real):
            _fail(f, "must be a number, got %r" % (state[f],))
    for f in ("filter_type", "mask_for_z"):
        if not isinstance(state[f], str):
            _fail(f, "must be a string, got %r" % (state[f],))
    if not isinstance(state["clean"], bool) or not isinstance(state["wide"], bool):
        _fail("clean", "and wide must be bools")
    vads = state["vads"]
    if vads is not None and not (isinstance(vads, (tuple, list)) and all(isinstance(v, str) for v in vads)):
        _fail("vads", "must be None or a pair of mask types")
    if vads is not None and not state["clean"]:
        _fail("clean", "must be True with vads")
    if state["kind"] != ("clean" if state["clean"] else "plain"):
        _fail("kind", "must be %r for clean=%r, got %r" % ("clean" if state["clean"] else "plain", state["clean"],
                                                             state["kind"]))
    try:
        _check_params(state["n_fft"], state["block"], state["lambda_cor"], state["lag"])
        check_opts(state["filter_type"], state["rank"], state["mask_for_z"], state["clean"], vads)
    except (TypeError, NotImplementedError, AttributeError, ValueError) as e:
        _fail("options", "are not those of a stream: %s" % e)


def check(state):
    """Validate a session state on the host; raises ValueError naming the first offending field."""
    from .stream import emission
    if not isinstance(state, dict):
        raise ValueError("session state: must be a dict, got %s" % type(state).__name__)
    if state.get("version") != VERSION:
        _fail("version", "%r is not known (this library reads version %d)" % (state.get("version"), VERSION))
    for k in KEYS:
        if k not in state:
            _fail(k, "is missing")
    _check_options(state)
    lay = _layout(state)
    K, B = lay.K, _int(state, "B", 1)
    if state["wide"] != (max(lay.channels) + K - 1 > 8):
        _fail("wide", "must be True exactly when C + K - 1 > 8")
    L, T, S, J = (_int(state, f) for f in COUNTERS)
    n_fft, P, lag = state["n_fft"], state["block"], state["lag"]
    if (T, S) != emission(L, n_fft):
        _fail("frames_out", "/ samples_out (%d, %d) do not match samples_in = %d: expected %r"
              % (T, S, L, emission(L, n_fft)))
    if J != T // P:
        _fail("closed", "must be frames_out // block = %d, got %d" % (T // P, J))
    F, H, nw = n_fft // 2 + 1, n_fft // 2, min(J, lag)
    clean, mode = state["clean"], state["mask_for_z"]
    groups = state["groups"]
    if not isinstance(groups, list) or len(groups) != len(lay.groups):
        _fail("groups", "must be a list of %d groups (one per channel count)" % len(lay.groups))
    for gi, (g, (C, nodes)) in enumerate(zip(groups, lay.groups)):
        name = lambda f: "groups[%d].%s" % (gi, f)
        if not isinstance(g, dict):
            _fail(name(""), "must be a dict")
        for k in GROUP_KEYS:
            if k not in g:
                _fail(name(k), "is missing")
        if g["C"] != C or list(g["nodes"]) != nodes:
            _fail(name("C"), "/ nodes must be %d / %r" % (C, nodes))
        n, D = len(nodes), C + K - 1
        _tensor(g["hist"], name("hist"), (B, n, C, n_fft), torch.float32)
        for f in ("hist_s", "hist_n"):
            _optional(g[f], name(f), (B, n, C, n_fft), torch.float32, clean)
        _tensor(g["Yblk"], name("Yblk"), (B, n, C, P, F), torch.complex64)
        for f in ("Sblk", "Nblk"):
            _optional(g[f], name(f), (B, n, C, P, F), torch.complex64, "use_oracle_" in mode)
        _pair(g["R1"], name("R1"), (B, n, F, C, C), J == 0)
        _pair(g["R2"], name("R2"), (B, n, F, D, D), J == 0)
        _tensor(g["W1"], name("W1"), (B, nw, n, F, C), torch.complex64)
        _tensor(g["W2"], name("W2"), (B, nw, n, F, D), torch.complex64)
    for f in ("m1", "m2"):
        _tensor(state[f], f, (B, K, P, F), torch.float32)
    _optional(state["zblk"], "zblk", (B, K, P, F), torch.complex64, K > 1)
    for f in ("zsblk", "znblk"):
        _optional(state[f], f, (B, K, P, F), torch.complex64, K > 1 and mode in ("compressed", "use_oracle_zs"))
    _tensor(state["carry"], "carry", (B, N_TIME if clean else 1, K, H), torch.float32)
    return state


def host(x):
    """A fresh contiguous host copy of device tensor x (None stays None)."""
    return None if x is None else torch.empty(x.shape, dtype=x.dtype).copy_(x.detach())


def settings(state):
    """The options, geometry and counters of a state: what states joined into one stream must share."""
    return {k: state[k] for k in OPTIONS + GEOMETRY + COUNTERS}


def concat(states):
    """One state of B = sum(B_i) streams from states of identical options, geometry and counters, in list order."""
    if isinstance(states, dict):
        states = [states]
    if not isinstance(states, (list, tuple)) or not states:
        raise ValueError("session state: expected a state or a non-empty list of states")
    for st in states:
        check(st)
    first = settings(states[0])
    for i, st in enumerate(states[1:], 1):
        for k, v in settings(st).items():
            if v != first[k]:
                _fail(k, "of state %d is %r, state 0 has %r: joined states must match" % (i, v, first[k]))
    if len(states) == 1:
        return states[0]
    cat = lambda xs: torch.cat([x.to(xs[0].device) for x in xs], 0)

    def cat_opt(xs):
        return None if xs[0] is None else cat(xs)

    def cat_pair(ps):
        """Carried matrices; a state still without them (closed = 0, no R0) joins as zeros: the scan's start."""
        if all(p is None for p in ps):
            return None
        like = next(p for p in ps if p is not None)
        B = lambda i: states[i]["B"]
        return [cat([torch.zeros((B(i),) + tuple(like[w].shape[1:]), dtype=like[w].dtype) if p is None else p[w]
                     for i, p in enumerate(ps)]) for w in range(2)]

    out = dict(states[0])
    out["B"] = sum(st["B"] for st in states)
    for f in ("m1", "m2", "carry"):
        out[f] = cat([st[f] for st in states])
    for f in ("zblk", "zsblk", "znblk"):
        out[f] = cat_opt([st[f] for st in states])
    out["groups"] = []
    for gi, g0 in enumerate(states[0]["groups"]):
        gs = [st["groups"][gi] for st in states]
        g = {"C": g0["C"], "nodes": list(g0["nodes"])}
        for f in ("hist", "Yblk", "W1", "W2"):
            g[f] = cat([x[f] for x in gs])
        for f in ("hist_s", "hist_n", "Sblk", "Nblk"):
            g[f] = cat_opt([x[f] for x in gs])
        for f in ("R1", "R2"):
            g[f] = cat_pair([x[f] for x in gs])
        out["groups"].append(g)
    return out


def nbytes(state):
    """The bytes of a state's tensors."""
    def walk(x):
        if isinstance(x, torch.Tensor):
            return x.numel() * x.element_size()
        if isinstance(x, dict):
            return sum(walk(v) for v in x.values())
        if isinstance(x, (list, tuple)):
            return sum(walk(v) for v in x)
        return 0
    return walk(state)
