"""Extent model of the C ABI (include/disco_b200.h): for every entry point that takes pointers, what each kernel
addresses behind each pointer, as a function of the call's scalar arguments.

ROWS[name][param] = (mode, dtype, count) with
  mode   'r' (read), 'w' (written), 'rw' (both), or 'host': a host int array the library reads before any launch
  dtype  the element type the kernel addresses: 'c64' (interleaved float2), 'f32', 'f64' or 'i32'
  count  a function of the call's arguments (a dict by parameter name) -> number of elements addressed

A device pointer must be aligned to its element size (float2 / double loads).  NULL pointers address nothing (the
library itself rejects a NULL where one is required).  Workspaces ('ws' dtype 'u8', counted in bytes) are sized
by the library's own size functions, which depend on disco_set_reserved_sms at the time of the call: `sizes` below
evaluates them.  The fused STFT kernel checks the 16-byte alignment its TMA loads of x need and falls back to plain
loads itself, so x carries no stricter requirement.

extents(name, args, sizes) evaluates one call; header_params() parses the header so that the CPU tests can require a
row for every pointer parameter of every declared entry point."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "disco_b200.h")
ITEMSIZE = {"c64": 8, "f32": 4, "f64": 8, "i32": 4, "u8": 1}


def F(a):
    return a["n_fft"] // 2 + 1


def n_frames(length, n_fft):
    return 1 + length // (n_fft // 2)


def T_of(a):
    return n_frames(a["length"], a["n_fft"])


def groups(a):
    """(utterance, node) groups of the concatenated-channel entry points (make_cat in csrc/api.cu)."""
    return a["n_utt"] * (a["n_sel"] if a.get("node_sel") else a["K"])


def D(a):
    return a["C"] + a["K"] - 1


def J(a):
    return -(-a["T"] // a["block"])


def _cat(extra):
    """Y and Z of the concatenated channel view, plus the node selection."""
    rows = {"Y": ("r", "c64", lambda a: groups(a) * a["C"] * a["T"] * F(a)),
            "Z": ("r", "c64", lambda a: a["n_utt"] * a["K"] * a["T"] * F(a)),
            "node_sel": ("host", "i32", lambda a: a["n_sel"])}
    rows.update(extra)
    return rows


# A workspace row's count is (kind, ...) instead of a function: ('stft', set count or the parameter holding it),
# ('bss',) or ('stoi',).  Its extent is what the library's size function asks for at the current reserved-SM
# setting, or the declared workspace_bytes if larger (the kernels trust that count).
_SCM2 = lambda a: groups(a) * F(a) * D(a) * D(a)
_PLANE_CAT = lambda a: groups(a) * a["T"] * F(a)

ROWS = {
    "disco_stft": {
        "x": ("r", "f32", lambda a: a["n_sig"] * a["length"]),
        "Y": ("w", "c64", lambda a: a["n_sig"] * T_of(a) * F(a))},
    "disco_stft_scm": {
        "x": ("r", "f32", lambda a: a["n_grp"] * a["C"] * a["length"]),
        "mask": ("r", "f32", lambda a: a["n_grp"] * T_of(a) * F(a)),
        "Y": ("w", "c64", lambda a: a["n_grp"] * a["C"] * T_of(a) * F(a)),
        "Rss": ("w", "c64", lambda a: a["n_grp"] * F(a) * a["C"] ** 2),
        "Rnn": ("w", "c64", lambda a: a["n_grp"] * F(a) * a["C"] ** 2),
        "workspace": ("w", "u8", ("stft", 1))},
    "disco_stft_scm2": {
        "x": ("r", "f32", lambda a: a["n_grp"] * a["C"] * a["length"]),
        "mask_a": ("r", "f32", lambda a: a["n_grp"] * T_of(a) * F(a)),
        "mask_b": ("r", "f32", lambda a: a["n_grp"] * T_of(a) * F(a)),
        "Y": ("w", "c64", lambda a: a["n_grp"] * a["C"] * T_of(a) * F(a)),
        "workspace": ("w", "u8", ("stft", 2))},
    "disco_stft_filter_dual": {
        "x": ("r", "f32", lambda a: a["n_grp"] * a["C"] * a["length"]),
        "W1": ("r", "c64", lambda a: a["n_grp"] * F(a) * a["C"]),
        "W2": ("r", "c64", lambda a: a["n_grp"] * F(a) * a["C"]),
        "z": ("w", "c64", lambda a: a["n_grp"] * T_of(a) * F(a)),
        "zn": ("w", "c64", lambda a: a["n_grp"] * T_of(a) * F(a)),
        "yf": ("w", "c64", lambda a: a["n_grp"] * T_of(a) * F(a))},
    "disco_scm_from_workspace": {
        "workspace": ("r", "u8", ("stft", "n_set")),
        "Rss": ("w", "c64", lambda a: a["n_grp"] * F(a) * a["C"] ** 2),
        "Rnn": ("w", "c64", lambda a: a["n_grp"] * F(a) * a["C"] ** 2)},
    "disco_tf_mask": {
        "S": ("r", "c64", lambda a: a["n_elem"]),
        "N": ("r", "c64", lambda a: a["n_elem"]),
        "M": ("w", "f32", lambda a: a["n_elem"])},
    "disco_masked_scm": _cat({
        "mask": ("r", "f32", _PLANE_CAT),
        "Rss": ("w", "c64", _SCM2),
        "Rnn": ("w", "c64", _SCM2)}),
    "disco_filter_sum_scm": {
        "W1": ("r", "c64", lambda a: a["n_grp"] * F(a) * a["C"]),
        "Y": ("r", "c64", lambda a: a["n_grp"] * a["C"] * a["T"] * F(a)),
        "mask": ("r", "f32", lambda a: a["n_grp"] * a["T"] * F(a)),
        "z_out": ("w", "c64", lambda a: a["n_grp"] * a["T"] * F(a)),
        "zn_out": ("w", "c64", lambda a: a["n_grp"] * a["T"] * F(a)),
        "Rss": ("w", "c64", lambda a: a["n_grp"] * F(a) * a["C"] ** 2),
        "Rnn": ("w", "c64", lambda a: a["n_grp"] * F(a) * a["C"] ** 2)},
    "disco_tango_mid": {
        "W1": ("r", "c64", lambda a: a["n_utt"] * a["K"] * F(a) * a["C"]),
        "Y": ("r", "c64", lambda a: a["n_utt"] * a["K"] * a["C"] * a["T"] * F(a)),
        "mask_w": ("r", "f32", lambda a: a["n_utt"] * a["K"] * a["T"] * F(a)),
        "Z": ("w", "c64", lambda a: a["n_utt"] * a["K"] * a["T"] * F(a)),
        "ZN": ("w", "c64", lambda a: a["n_utt"] * a["K"] * a["T"] * F(a)),
        "Rss": ("w", "c64", lambda a: a["n_utt"] * a["K"] * F(a) * D(a) ** 2),
        "Rnn": ("w", "c64", lambda a: a["n_utt"] * a["K"] * F(a) * D(a) ** 2)},
    "disco_mwf_solve": {
        "Rss": ("r", "c64", lambda a: a["n_mat"] * a["D"] ** 2),
        "Rnn": ("r", "c64", lambda a: a["n_mat"] * a["D"] ** 2),
        "W": ("w", "c64", lambda a: a["n_mat"] * a["D"]),
        "T1": ("w", "c64", lambda a: a["n_mat"] * a["D"])},
    "disco_mwf_solve_workspace": {
        "workspace": ("r", "u8", ("stft", 1)),
        "W": ("w", "c64", lambda a: a["n_grp"] * F(a) * a["C"]),
        "T1": ("w", "c64", lambda a: a["n_grp"] * F(a) * a["C"]),
        "Rss": ("w", "c64", lambda a: a["n_grp"] * F(a) * a["C"] ** 2),
        "Rnn": ("w", "c64", lambda a: a["n_grp"] * F(a) * a["C"] ** 2)},
    "disco_mwf_solve_workspace2": {
        "workspace": ("r", "u8", ("stft", 2)),
        "W": ("w", "c64", lambda a: 2 * a["n_grp"] * F(a) * a["C"]),
        "T1": ("w", "c64", lambda a: 2 * a["n_grp"] * F(a) * a["C"])},
    "disco_filter_sum": _cat({
        "W": ("r", "c64", lambda a: groups(a) * F(a) * D(a)),
        "out": ("w", "c64", _PLANE_CAT),
        "resid": ("w", "c64", _PLANE_CAT)}),
    "disco_filter_dual": {
        "W1": ("r", "c64", lambda a: a["n_grp"] * F(a) * a["C"]),
        "W2": ("r", "c64", lambda a: a["n_grp"] * F(a) * a["C"]),
        "Y": ("r", "c64", lambda a: a["n_grp"] * a["C"] * a["T"] * F(a)),
        "z": ("w", "c64", lambda a: a["n_grp"] * a["T"] * F(a)),
        "zn": ("w", "c64", lambda a: a["n_grp"] * a["T"] * F(a)),
        "yf": ("w", "c64", lambda a: a["n_grp"] * a["T"] * F(a))},
    "disco_istft": {
        "Y": ("r", "c64", lambda a: a["n_sig"] * a["T"] * F(a)),
        "x": ("w", "f32", lambda a: a["n_sig"] * a["length"])},
    "disco_stft_lengths": {
        "x": ("r", "f32", lambda a: a["n_sig"] * a["length"]),
        "lengths": ("r", "i32", lambda a: a["n_sig"]),
        "lengths_host": ("host", "i32", lambda a: a["n_sig"]),
        "Y": ("w", "c64", lambda a: a["n_sig"] * T_of(a) * F(a))},
    "disco_istft_lengths": {
        "Y": ("r", "c64", lambda a: a["n_sig"] * a["T"] * F(a)),
        "lengths": ("r", "i32", lambda a: a["n_sig"]),
        "lengths_host": ("host", "i32", lambda a: a["n_sig"]),
        "x": ("w", "f32", lambda a: a["n_sig"] * a["length"])},
    "disco_stream_stft": {
        "hist": ("r", "f32", lambda a: a["n_sig"] * a["n_fft"]),
        "chunk": ("r", "f32", lambda a: a["n_sig"] * a["n_new"]),
        "hist_out": ("w", "f32", lambda a: a["n_sig"] * a["n_fft"]),
        "Y": ("w", "c64", lambda a: a["n_sig"] * a["n_fr"] * F(a)),
        "Y_blk": ("w", "c64", lambda a: a["n_sig"] * a["blk_frames"] * F(a))},
    "disco_stream_istft": {
        "Y": ("r", "c64", lambda a: a["n_sig"] * a["n_fr"] * F(a)),
        "carry": ("rw", "f32", lambda a: a["n_sig"] * (a["n_fft"] // 2)),
        "x": ("w", "f32", lambda a: a["n_sig"] * a["x_stride"])},
    "disco_stream_stft_slots": {
        "hist": ("rw", "f32", lambda a: 2 * a["n_slot"] * a["n_sig"] * a["n_fft"]),
        "chunk": ("r", "f32", lambda a: a["n_slot"] * a["n_sig"] * a["n_max"]),
        "Y": ("w", "c64", lambda a: a["n_slot"] * a["n_sig"] * a["f_max"] * F(a)),
        "Y_blk": ("w", "c64", lambda a: a["n_slot"] * a["n_sig"] * a["blk_frames"] * F(a)),
        "slots": ("r", "i32", lambda a: a["n_slot"] * 8),
        "slots_host": ("host", "i32", lambda a: a["n_slot"] * 8)},
    "disco_stream_istft_slots": {
        "Y": ("r", "c64", lambda a: a["n_slot"] * a["n_sig"] * a["f_max"] * F(a)),
        "carry": ("rw", "f32", lambda a: a["n_slot"] * a["n_sig"] * (a["n_fft"] // 2)),
        "x": ("w", "f32", lambda a: a["n_slot"] * a["n_sig"] * a["s_max"]),
        "slots": ("r", "i32", lambda a: a["n_slot"] * 5),
        "slots_host": ("host", "i32", lambda a: a["n_slot"] * 5)},
    "disco_band_stats": {
        "x": ("r", "f32", lambda a: (a["n_sig"] - 1) * a["row_stride"] + a["length"]),
        "sel": ("r", "f32", lambda a: (a["n_sig"] - 1) * a["row_stride"] + a["length"]),
        "ba": ("r", "f64", lambda a: a["n_band"] * 2 * (a["order"] + 1)),
        "stats": ("w", "f64", lambda a: a["n_sig"] * a["n_band"] * 3)},
    "disco_bss_eval": {
        "refs": ("r", "f32", lambda a: a["n_set"] * a["nsrc"] * a["length"]),
        "ests": ("r", "f32", lambda a: a["n_set"] * a["n_est"] * a["length"]),
        "norms": ("w", "f64", lambda a: a["n_set"] * a["n_est"] * (1 + 2 * a["nsrc"])),
        "workspace": ("w", "u8", ("bss",))},
    "disco_resample_poly": {
        "x": ("r", "f32", lambda a: a["n_sig"] * a["length"]),
        "y": ("w", "f64", lambda a: a["n_sig"] * -(-a["length"] * a["up"] // a["down"])),
        "taps": ("r", "f64", lambda a: a["n_taps"])},
    "disco_stoi": {
        "cleans": ("r", "f64", lambda a: a["n_clean"] * a["length"]),
        "degraded": ("r", "f64", lambda a: a["n_deg"] * a["length"]),
        "pairs": ("r", "i32", lambda a: a["n_pair"] * 2),
        "d": ("w", "f64", lambda a: a["n_pair"]),
        "n_sel": ("w", "i32", lambda a: a["n_clean"]),
        "n_frames": ("w", "i32", lambda a: a["n_pair"]),
        "workspace": ("w", "u8", ("stoi",))},
    "disco_transpose_c64": {
        "in": ("r", "c64", lambda a: a["batch"] * a["rows"] * a["cols"]),
        "out": ("w", "c64", lambda a: a["batch"] * a["rows"] * a["cols"])},
    "disco_transpose_f32": {
        "in": ("r", "f32", lambda a: a["batch"] * a["rows"] * a["cols"]),
        "out": ("w", "f32", lambda a: a["batch"] * a["rows"] * a["cols"])},
    "disco_apply_mask": {
        "in": ("r", "c64", lambda a: a["n_elem"]),
        "m": ("r", "f32", lambda a: a["n_elem"]),
        "out": ("w", "c64", lambda a: a["n_elem"])},
    "disco_apply_mask_channels": {
        "in": ("r", "c64", lambda a: a["n_grp"] * a["chans"] * a["plane"]),
        "m": ("r", "f32", lambda a: a["n_grp"] * a["plane"]),
        "out": ("w", "c64", lambda a: a["n_grp"] * a["chans"] * a["plane"])},
}

_REC = {
    "R0ss": ("r", "c64", _SCM2),
    "R0nn": ("r", "c64", _SCM2),
    "Rss": ("w", "c64", lambda a: groups(a) * J(a) * F(a) * D(a) ** 2),
    "Rnn": ("w", "c64", lambda a: groups(a) * J(a) * F(a) * D(a) ** 2),
    "mask": ("r", "f32", _PLANE_CAT)}
_BLK = {
    "W": ("r", "c64", lambda a: groups(a) * J(a) * F(a) * D(a)),
    "out": ("w", "c64", _PLANE_CAT),
    "resid": ("w", "c64", _PLANE_CAT)}
_FRAMES = {"frames": ("r", "i32", lambda a: a["n_utt"]),
           "frames_host": ("host", "i32", lambda a: a["n_utt"])}
ROWS["disco_scm_recursive"] = _cat(_REC)
ROWS["disco_scm_recursive_lengths"] = _cat(dict(_REC, **_FRAMES))
ROWS["disco_filter_sum_blocks"] = _cat(_BLK)
ROWS["disco_filter_sum_blocks_lengths"] = _cat(dict(_BLK, **_FRAMES))
ROWS["disco_resample_poly_lengths"] = dict(ROWS["disco_resample_poly"],
                                           lengths=("r", "i32", lambda a: a["n_sig"]),
                                           lengths_host=("host", "i32", lambda a: a["n_sig"]))
ROWS["disco_stoi_lengths"] = dict(ROWS["disco_stoi"],
                                  lengths=("r", "i32", lambda a: a["n_clean"]),
                                  lengths_host=("host", "i32", lambda a: a["n_clean"]))

# The workspaces the fused STFT+SCM kernels write and the consumers read: (producer, set count)
WS_PRODUCERS = {"disco_stft_scm": 1, "disco_stft_scm2": 2}
WS_CONSUMERS = {"disco_mwf_solve_workspace": 1, "disco_mwf_solve_workspace2": 2, "disco_scm_from_workspace": "n_set"}


def header_params():
    """{entry point: [(C type, parameter name)]} of every DISCO_API function the header declares."""
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    out = {}
    for m in re.finditer(r"DISCO_API\s+[\w\s\*]+?\b(disco_\w+)\s*\(([^)]*)\)", src):
        params = []
        for p in m.group(2).split(","):
            p = " ".join(p.split())
            if not p or p == "void":
                continue
            tm = re.match(r"(.*?[\s\*])(\w+)$", p)
            params.append((tm.group(1).strip(), tm.group(2)))
        out[m.group(1)] = params
    return out


def pointer_params(params):
    """The pointer parameters of one entry point, without the stream."""
    return [n for t, n in params if "*" in t and n != "stream"]


class Extent:
    __slots__ = ("param", "mode", "dtype", "nbytes", "count")

    def __init__(self, param, mode, dtype, count):
        self.param, self.mode, self.dtype, self.count = param, mode, dtype, int(count)
        self.nbytes = max(self.count, 0) * ITEMSIZE[dtype]

    def __repr__(self):
        return "%s %s %s x %d (%d bytes)" % (self.param, self.mode, self.dtype, self.count, self.nbytes)


def extents(name, args, sizes):
    """The extents of one call of `name`.  args: {parameter: value}, with pointer parameters truthy when non-NULL;
    sizes: object with stft_ws(n_grp, C, length, n_fft, n_set), bss_ws(n_set, nsrc, n_est, length, flen) and
    stoi_ws(n_clean, n_pair, length), the library's size functions at the current setting."""
    out = []
    for param, (mode, dtype, count) in ROWS[name].items():
        if not args.get(param):
            continue
        if isinstance(count, tuple):
            kind = count[0]
            a = args
            if kind == "stft":
                n_set = a[count[1]] if isinstance(count[1], str) else count[1]
                need = sizes.stft_ws(a["n_grp"], a["C"], a["length"], a["n_fft"], n_set)
            elif kind == "bss":
                need = sizes.bss_ws(a["n_set"], a["nsrc"], a["n_est"], a["length"], a["flen"])
            else:
                need = sizes.stoi_ws(a["n_clean"], a["n_pair"], a["length"])
            n = max(int(need), int(a.get("workspace_bytes", 0)))
        else:
            n = count(args)
        out.append(Extent(param, mode, dtype, n))
    return out


class Refused(Exception):
    """A call the model refuses: it is never forwarded to the library."""


class Span:
    """What a registered device buffer covers: base address, bytes, dtype name, device index, whether it is dense."""
    __slots__ = ("addr", "nbytes", "dtype", "device", "owner", "contiguous")

    def __init__(self, addr, nbytes, dtype, device, owner=None, contiguous=True):
        self.addr, self.nbytes, self.dtype, self.device, self.owner = addr, nbytes, dtype, device, owner
        self.contiguous = contiguous


def check_call(name, args, lookup, sizes, device, host_len):
    """Evaluate one call against the model; raises Refused on the first violation.
    lookup(addr) -> Span registered at that address (or None); host_len(value) -> element count and dtype of a host
    array argument; device: the index of the current device."""
    for e in extents(name, args, sizes):
        v = args[e.param]
        if e.mode == "host":
            n, dt = host_len(v)
            if dt != "i32" or n != e.count:
                raise Refused("%s: host array %s holds %d %s, the call declares %d" % (name, e.param, n, dt, e.count))
            continue
        sp = lookup(v)
        if sp is None:
            raise Refused("%s: %s = 0x%x is not a tensor handed to the library" % (name, e.param, v))
        if sp.device != device:
            raise Refused("%s: %s lives on %s, the call runs on cuda:%d" % (
                name, e.param, sp.device if sp.device == "cpu" else "cuda:%s" % sp.device, device))
        if e.dtype != "u8" and sp.dtype != e.dtype:
            raise Refused("%s: %s is %s, the kernel addresses %s" % (name, e.param, sp.dtype, e.dtype))
        if v % ITEMSIZE[e.dtype]:
            raise Refused("%s: %s = 0x%x is not %d-byte aligned" % (name, e.param, v, ITEMSIZE[e.dtype]))
        if e.nbytes > sp.nbytes:
            raise Refused("%s: %s %s past the end of its tensor: %d bytes addressed, %d held"
                          % (name, e.param, "reads" if e.mode == "r" else "writes", e.nbytes, sp.nbytes))
