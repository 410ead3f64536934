"""Every route of Tango's batched layer, under every filter setting and non-default options, against float64 with a
complex metric.

`tango_batched` picks one of several kernel chains (tango.py: fuse_dual, same_mask, fuse_mid, fuse_multi, the generic
step 2, the exchange modes, a callable step-2 mask, and the ragged `offline_tango` adapter), and `tango_step1` one of
three sub-routes (S1a: fused STFT+SCM with the workspace solve, C <= 4; S1b: fused with the matrices materialised,
C 5..8; S1c: unfused).  `ref_mic`, `mu`, `filter_type` and `rank` are forwarded separately at every call site, so a
dropped argument silently gives the default on one route only.  ROUTES states, per row, the inputs that select a route
and the `ops` call sites it must and must not reach; tests/test_tango_routes_cpu.py parses the call sites out of the
sources and fails on CPU when one is named by no row.

Each (row, filter setting) case checks:
1. spy: the call sites reached, and the `ref` / `mu` / `type` / `rank` every call received;
2. masks: masks_z bit-equal to ops.tf_mask of microphone ref_mic of ops.stft(s), mask_w of microphone 0 (or mask_z
   itself where the route reuses it), external masks returned unchanged, a callable mask_w fed the route's Y, z_y, zn;
3. values: every complex output per (utterance, node) within conftest.TOL complex relative L2 of float64 (tango_f64
   where it states the mode, tango_np(double=True) elsewhere; the record_parity fallback where the fp32 port is itself
   >= TOL from float64), recorded as a complex and a magnitude row;
4. zn = Y[ref] - z_y entry-wise to one rounding, Y the spectrum the route used (the STFT bound for fuse_dual, which
   never stores Y);
5. FT outputs = transposed TF outputs (bit for bit, or within the filter bound where the layouts run different filter
   kernels), and yf, z_y, zn bit-identical with and without diagnostics;
6. discrimination: the float64 oracle at each neighbouring option (ref_mic 0 <-> C-1, mu 1 <-> 2.5, rank 1 <-> 2,
   gevd <-> mwf) lies more than 10x the case's bar from the true one on some compared output, and the checker rejects
   conj(yf), -zn and yf with the two masks swapped.
`online_tango` is checked the same way at non-default ref_mic, rank, lag, block and R0 against the per-frame float64
composition of oracle/online_np.
"""
import ast
import inspect
import math
import os
import sys

import numpy as np
import pytest
import torch

from conftest import TOL, record_parity, rel_l2, rel_l2_mag

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "disco_b200")
U = 2.0 ** -24
# the filter settings of tests/test_gpu_solver_edges.py: (type, rank, mu)
FILTERS = [("gevd", 1, 1.0), ("gevd", 2, 2.5), ("gevd", "full", 1.0), ("r1-mwf", 1, 2.5), ("mwf", 1, 1.0)]

# ---- call sites ---------------------------------------------------------------------------------------------------
# the functions whose `ops.<name>(` calls the table must cover, and the ops that only compute on the host
SITE_FUNCS = {"tango.py": ("tango_batched", "tango_step1", "tango_step2", "_z_for_stats", "_offline_tango_ragged"),
              "online.py": ("online_mwf", "online_tango")}
HOST_OPS = {"n_frames", "_layout", "stft_scm_supported", "tango_mid_supported", "signal_lengths"}
# sites no row here reaches, with the tests that do
EXEMPT = {"tango_batched:stft_lengths": "uneven lengths= batches: tests/test_gpu_lengths.py",
          "tango_step1:stft_lengths": "uneven lengths= batches: tests/test_gpu_lengths.py",
          "_offline_tango_ragged:stft#3": "network step-1 masks of a ragged array: tests/test_dnn_mask.py"}


def call_sites():
    """{site: (file, line, col)} of every `ops.<name>(` call inside SITE_FUNCS (lambdas included), host ops excluded.
    site = 'function:op', or 'function:op#i' (i-th in source order) where the function calls op more than once."""
    found = {}
    for fname, funcs in SITE_FUNCS.items():
        path = os.path.join(PKG, fname)
        with open(path) as fh:
            tree = ast.parse(fh.read())
        for fn in (n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in funcs):
            calls = sorted(((c.lineno, c.col_offset, c.func.attr) for c in ast.walk(fn)
                            if isinstance(c, ast.Call) and isinstance(c.func, ast.Attribute)
                            and isinstance(c.func.value, ast.Name) and c.func.value.id == "ops"
                            and c.func.attr not in HOST_OPS))
            names = [op for _, _, op in calls]
            seen = {}
            for line, col, op in calls:
                seen[op] = seen.get(op, 0) + 1
                site = "%s:%s" % (fn.name, op) + ("#%d" % seen[op] if names.count(op) > 1 else "")
                found[site] = (path, line, col)
    return found


# ---- the route table ----------------------------------------------------------------------------------------------
S1A = ("tango_step1:stft_scm#1", "tango_step1:mwf_solve_workspace")
S1B = ("tango_step1:stft_scm#2", "tango_step1:mwf_solve")
S1C = ("tango_step1:stft", "tango_step1:masked_scm#1", "tango_step1:mwf_solve")
S1_ORACLE = ("tango_step1:stft", "tango_step1:masked_scm#2", "tango_step1:masked_scm#3", "tango_step1:mwf_solve",
             "tango_step1:filter_sum#2")
S1A_F, S1B_F, S1C_F = S1A + ("tango_step1:filter_sum#1",), S1B + ("tango_step1:filter_sum#2",), \
    S1C + ("tango_step1:filter_sum#2",)
STEP1 = tuple(sorted(set(S1A_F + S1B_F + S1C_F + S1_ORACLE)))
T2_LOCAL = ("tango_step2:masked_scm#1", "tango_step2:mwf_solve", "tango_step2:filter_sum")
T2_EXCH = ("tango_step2:masked_scm#2", "tango_step2:masked_scm#3", "tango_step2:mwf_solve", "tango_step2:filter_sum")
STEP2 = tuple(sorted(set(T2_LOCAL + T2_EXCH)))
NOT_LOCAL2 = ("tango_step2:masked_scm#1",)        # the step-2 statistics of 'local'
# the clean spectra and the diagnostic outputs z_s, z_n, sf, nf (s and n are always given here)
DIAG = ("tango_batched:stft", "tango_batched:filter_sum#1", "tango_batched:filter_sum#2", "tango_batched:filter_sum#4",
        "tango_batched:filter_sum#5")
DUAL = ("tango_batched:stft_scm2", "tango_batched:mwf_solve_workspace2", "tango_batched:stft_filter_dual")
MID = ("tango_batched:filter_sum_scm",)
MULTI = ("tango_batched:tango_mid",)
R2 = ("tango_batched:mwf_solve", "tango_batched:filter_sum#3")
DISTANT = ("_z_for_stats:apply_mask#1", "_z_for_stats:apply_mask#2")
COMPRESSED = ("_z_for_stats:tf_mask", "_z_for_stats:apply_mask#3", "_z_for_stats:apply_mask#4")
RAGGED = ("_offline_tango_ragged:stft#1", "_offline_tango_ragged:stft#2", "_offline_tango_ragged:filter_sum#1",
          "_offline_tango_ragged:filter_sum#2", "_offline_tango_ragged:filter_sum#3",
          "_offline_tango_ragged:filter_sum#4", "_offline_tango_ragged:transpose_last2")
ONLINE_SITES = ("online_tango:stft", "online_mwf:scm_recursive", "online_mwf:mwf_solve", "online_mwf:filter_sum_blocks")


def _row(id, route, K, C, n_fft, masks, ref, calls, never, vads=("irm1", "irm2"), mfz="local", B=1, chans=None):
    """masks: 'oracle' (vads of s, n), 'external' (two random masks), 'same' (masks=(mz, None)), 'callable' (a step-2
    estimator on Y, z_y, zn; mask_z alternates oracle / external) or 'alt' (oracle for even filter settings, external
    for odd); ref: 0, 'last' (C - 1) or 'alt' (0 for even filter settings, C - 1 for odd)."""
    return dict(id=id, route=route, K=K, C=C, n_fft=n_fft, masks=masks, ref=ref, calls=tuple(calls),
                never=tuple(never), vads=vads, mfz=mfz, B=B, chans=chans)


_NOT_FUSED2 = DUAL + MID + MULTI + R2
ROUTES = [
    # fuse_dual: K = 1, local, two different masks, C <= 4, n_fft 256 / 512
    _row("dual_c1", "fuse_dual", 1, 1, 256, "alt", 0, DUAL + DIAG, STEP1 + STEP2 + MID + MULTI + R2, B=2),
    _row("dual_c4_512", "fuse_dual", 1, 4, 512, "alt", "alt", DUAL + DIAG, STEP1 + STEP2 + MID + MULTI + R2),
    _row("dual_c3", "fuse_dual", 1, 3, 256, "external", "last", DUAL + DIAG, STEP1 + STEP2 + MID + MULTI + R2, B=2),
    _row("dual_c4_eqvad_last", "fuse_dual", 1, 4, 256, "oracle", "last", DUAL + DIAG,
         STEP1 + STEP2 + MID + MULTI + R2, vads=("irm1", "irm1")),
    # same_mask: K = 1 and mask_w is mask_z
    _row("same_c4", "same_mask", 1, 4, 512, "oracle", 0, S1A_F + DIAG, _NOT_FUSED2 + STEP2, vads=("irm1", "irm1")),
    _row("same_c6", "same_mask", 1, 6, 512, "same", "alt", S1B_F + DIAG, _NOT_FUSED2 + STEP2),
    _row("same_c10", "same_mask", 1, 10, 256, "same", "alt", S1C_F + DIAG, _NOT_FUSED2 + STEP2),
    # fuse_mid: K = 1, different masks, no fuse_dual, C <= 8
    _row("mid_c6_512", "fuse_mid", 1, 6, 512, "alt", "alt", S1B + MID + R2 + DIAG, DUAL + MULTI + STEP2 +
         ("tango_step1:filter_sum#1", "tango_step1:filter_sum#2")),
    _row("mid_c3_1024", "fuse_mid", 1, 3, 1024, "external", "last", S1A + MID + R2 + DIAG, DUAL + MULTI + STEP2 +
         ("tango_step1:filter_sum#1", "tango_step1:filter_sum#2")),
    _row("mid_c7_1024", "fuse_mid", 1, 7, 1024, "oracle", "alt", S1C + MID + R2 + DIAG, DUAL + MULTI + STEP2 +
         ("tango_step1:filter_sum#1", "tango_step1:filter_sum#2"), vads=("irm2", "irm1")),
    # K = 1 generic: C 9..16
    _row("k1_generic_c12", "k1_generic", 1, 12, 256, "alt", "alt", S1C_F + T2_LOCAL + DIAG, _NOT_FUSED2),
    # fuse_multi: K > 1, local, tango_mid_supported
    _row("multi_c2k3", "fuse_multi", 3, 2, 256, "alt", "alt", S1A + MULTI + R2 + DIAG, DUAL + MID + STEP2 +
         ("tango_step1:filter_sum#1",)),
    _row("multi_c1k4", "fuse_multi", 4, 1, 512, "external", 0, S1A + MULTI + R2 + DIAG, DUAL + MID + STEP2 +
         ("tango_step1:filter_sum#1",)),
    _row("multi_c4k2", "fuse_multi", 2, 4, 1024, "oracle", "last", S1A + MULTI + R2 + DIAG, DUAL + MID + STEP2 +
         ("tango_step1:filter_sum#1",)),
    # K > 1 generic: (C, K) tango_mid does not support
    _row("kgen_c5k2", "k_generic", 2, 5, 512, "alt", "alt", S1B_F + T2_LOCAL + DIAG, _NOT_FUSED2),
    _row("kgen_c2k5", "k_generic", 5, 2, 256, "alt", "last", S1A_F + T2_LOCAL + DIAG, _NOT_FUSED2),
    # exchange modes at (C, K) = (2, 3)
    _row("x_distant", "exchange", 3, 2, 256, "alt", "alt", S1A_F + DISTANT + T2_EXCH + DIAG, _NOT_FUSED2 + NOT_LOCAL2,
         mfz="distant"),
    _row("x_compressed", "exchange", 3, 2, 256, "alt", "alt", S1A_F + COMPRESSED + T2_EXCH + DIAG,
         _NOT_FUSED2 + NOT_LOCAL2, mfz="compressed"),
    _row("x_oracle_refs", "exchange", 3, 2, 256, "alt", "alt", S1_ORACLE + T2_EXCH + DIAG,
         _NOT_FUSED2 + NOT_LOCAL2 + S1A, mfz="use_oracle_refs"),
    _row("x_oracle_zs", "exchange", 3, 2, 256, "alt", "alt", S1_ORACLE + T2_EXCH + DIAG, _NOT_FUSED2 + NOT_LOCAL2 + S1A,
         mfz="use_oracle_zs"),
    _row("x_previous", "exchange", 3, 2, 256, "alt", "alt", S1A_F + T2_EXCH + DIAG, _NOT_FUSED2 + NOT_LOCAL2 + DISTANT,
         mfz="previous"),
    # a callable step-2 mask estimator
    _row("est_k1c4", "estimator", 1, 4, 512, "callable", "alt", S1A_F + T2_LOCAL + DIAG, _NOT_FUSED2),
    _row("est_k3c2", "estimator", 3, 2, 256, "callable", "alt", S1A_F + T2_LOCAL + DIAG, _NOT_FUSED2),
    # the reference-signature adapter on nodes of different microphone counts (its reference microphone is 0)
    _row("ragged_local", "ragged", 3, 3, 256, "alt", 0, RAGGED + S1A_F + T2_LOCAL, _NOT_FUSED2, chans=[2, 3, 2]),
    _row("ragged_compressed", "ragged", 3, 3, 256, "alt", 0, RAGGED + S1A_F + COMPRESSED + T2_EXCH,
         _NOT_FUSED2 + NOT_LOCAL2, chans=[2, 3, 2], mfz="compressed"),
]

# online_tango: (K, C), options; n_fft cycles 256 / 512 / 1024
ONLINE = [
    dict(id="on_k1c4", K=1, C=4, n_fft=256, ref="last", rank=1, lag=1, block=4, R0=True, calls=ONLINE_SITES),
    dict(id="on_k1c4_l0", K=1, C=4, n_fft=1024, ref=0, rank=2, lag=0, block=16, R0=False, calls=ONLINE_SITES),
    dict(id="on_k2c3", K=2, C=3, n_fft=512, ref="last", rank=2, lag=2, block=4, R0=True, calls=ONLINE_SITES),
    dict(id="on_k2c3_b16", K=2, C=3, n_fft=256, ref=0, rank=1, lag=1, block=16, R0=False, calls=ONLINE_SITES),
    dict(id="on_k1c12", K=1, C=12, n_fft=512, ref="last", rank=2, lag=1, block=16, R0=True, calls=ONLINE_SITES),
    dict(id="on_k1c12_r0", K=1, C=12, n_fft=256, ref=0, rank=1, lag=2, block=4, R0=False, calls=ONLINE_SITES),
    dict(id="on_k4c6", K=4, C=6, n_fft=256, ref="last", rank=1, lag=1, block=4, R0=True, calls=ONLINE_SITES),
    dict(id="on_k4c6_lag0", K=4, C=6, n_fft=512, ref=0, rank=2, lag=0, block=16, R0=False, calls=ONLINE_SITES),
]


def case_options(row, fi):
    """(type, rank, mu, ref_mic, mask kind, primary layout) of row under filter setting fi."""
    typ, rank, mu = FILTERS[fi]
    C = row["C"]
    ref = {0: 0, "last": C - 1, "alt": (C - 1) * (fi % 2)}[row["ref"]]
    kind = row["masks"] if row["masks"] != "alt" else ("oracle", "external")[fi % 2]
    layout = ("FT", "TF")[fi % 2]
    return typ, rank, mu, ref, kind, layout


# ---- spy on the ops that tango.py / online.py call ------------------------------------------------------------------
SPIED = ("stft", "stft_lengths", "stft_scm", "stft_scm2", "mwf_solve_workspace", "mwf_solve_workspace2",
         "stft_filter_dual", "filter_sum", "filter_sum_scm", "tango_mid", "masked_scm", "mwf_solve", "apply_mask",
         "tf_mask", "transpose_last2", "scm_recursive", "filter_sum_blocks")
_SITES = None


def _site_index():
    global _SITES
    if _SITES is None:
        _SITES = {}
        for site, (path, line, col) in call_sites().items():
            _SITES[(path, line, col)] = site
    return _SITES


class Spy:
    """Records every spied ops call made from tango.py / online.py: (site or None for a helper, bound arguments with
    defaults, return value)."""

    def __init__(self, monkeypatch):
        from disco_b200 import ops
        self.calls = []
        index = _site_index()
        files = {os.path.join(PKG, f) for f in SITE_FUNCS}
        for name in SPIED:
            orig = getattr(ops, name)
            sig = inspect.signature(orig)

            def wrap(*a, _orig=orig, _sig=sig, _name=name, **kw):
                fr = sys._getframe(1)
                path = os.path.abspath(fr.f_code.co_filename)
                out = _orig(*a, **kw)
                if path in files or os.path.dirname(path) == PKG:
                    site = None
                    if path in files:
                        pos = list(fr.f_code.co_positions())[fr.f_lasti // 2]
                        site = index.get((path, pos[0], pos[2]))
                        if site is None:
                            on_line = [s for (p, ln, _), s in index.items() if p == path and ln == pos[0]
                                       and s.split(":")[1].split("#")[0] == _name]
                            site = on_line[0] if len(on_line) == 1 else None
                    b = _sig.bind(*a, **kw)
                    b.apply_defaults()
                    self.calls.append((site, _name, dict(b.arguments), out))
                return out
            monkeypatch.setattr(ops, name, wrap)

    def clear(self):
        self.calls = []

    def sites(self):
        return {s for s, _, _, _ in self.calls if s is not None}

    def of(self, site):
        return [(args, out) for s, _, args, out in self.calls if s == site]

    def check_options(self, typ, rank, mu, ref, what):
        for site, name, args, _ in self.calls:
            if name in ("mwf_solve", "mwf_solve_workspace", "mwf_solve_workspace2"):
                got = (args["type"], args["rank"], float(args["mu"]))
                assert got == (typ, rank, float(mu)), "%s: %s (%s) received type/rank/mu %s" % (what, site, name, got)
            if name in ("stft_filter_dual", "filter_sum_scm", "tango_mid", "filter_sum_blocks") or \
                    (name == "filter_sum" and args["ref"] is not None):
                assert int(args["ref"]) == ref, "%s: %s (%s) received ref %s, case ref_mic %d" % (
                    what, site, name, args["ref"], ref)


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


# ---- inputs and oracles -----------------------------------------------------------------------------------------------
def case_length(row):
    """About 1 s, more where 10 D frames need it (D = C + K - 1 of step 2)."""
    hop = row["n_fft"] // 2
    D = row["C"] + row["K"] - 1
    return max(16000, hop * 10 * D + hop)


def _oracle_masks_f64(s, n, vads, ref, n_fft):
    """float64 step-1 / step-2 oracle masks (K, F, T) of one utterance (s, n of (K, C, L)): vads[0] of microphone ref,
    vads[1] of microphone 0 (mask_z itself for the same type with ref = 0)."""
    from oracle import tango_f64
    st = lambda x: np.array([tango_f64.stft64(c, n_fft, n_fft // 2) for c in x])
    mz = tango_f64.irm(st(s[:, ref]), st(n[:, ref]), int(vads[0][-1]))
    if vads[1] == vads[0] and ref == 0:
        return mz, mz
    return mz, tango_f64.irm(st(s[:, 0]), st(n[:, 0]), int(vads[1][-1]))


def f64_oracle(row, y, s, n, masks, vads, ref, typ, rank, mu, mfz, double_port=False):
    """The yardstick of one utterance: dict of (K, F, T) outputs.  masks: (mz, mw) (K, F, T) arrays, or None for the
    oracle vads.  tango_f64 where it states the mode (uniform arrays, 'local' / 'distant'), tango_np(double=True)
    elsewhere; double_port=False gives the fp32 port (tango_np, single precision) instead."""
    from oracle import tango_f64, tango_np
    n_fft = row["n_fft"]
    names = ("yf", "sf", "nf", "z_y", "z_s", "z_n", "zn", "masks_z", "mask_w")
    ragged = row["chans"] is not None
    if not double_port or ragged or mfz not in ("local", "distant"):
        ml = None if masks is None else ([m for m in masks[0]], [m for m in masks[1]])
        res = tango_np.offline_tango(y, s, n, vads=vads, mask_for_z=mfz, n_fft=n_fft, n_hop=n_fft // 2, mu=mu,
                                     filter_type=typ, rank=rank, ref_mic=ref, granularity="bin", masks=ml,
                                     double=double_port)
        return {k: np.array(v) for k, v in zip(names, res) if v is not None}
    if masks is None:
        masks = _oracle_masks_f64(np.asarray(s), np.asarray(n), vads, ref, n_fft)
    return tango_f64.offline_tango(np.asarray(y), np.asarray(s), np.asarray(n), masks=masks, n_fft=n_fft,
                                   n_hop=n_fft // 2, mu=mu, filter_type=typ, rank=rank, mask_for_z=mfz, ref_mic=ref)


def _ft(a):
    """[..., T, F] torch -> [..., F, T] numpy."""
    return a.transpose(-1, -2).cpu().numpy()


def _neighbours(typ, rank, mu, ref, C, D_max):
    """The options one step away from the case's, each as (label, typ, rank, mu, ref); inert ones left out (D = 1:
    every filter is lambda / (lambda + mu), so rank does not matter and gevd at mu 1 equals mwf)."""
    out = []
    if C > 1:
        out.append(("ref_mic", typ, rank, mu, C - 1 if ref == 0 else 0))
    if typ in ("gevd", "r1-mwf"):
        out.append(("mu", typ, rank, 2.5 if mu == 1.0 else 1.0, ref))
    if typ == "gevd" and D_max > 1:
        out.append(("rank", typ, {1: 2, 2: 1, "full": 1}[rank], mu, ref))
    if not (D_max == 1 and mu == 1.0):
        # the full-rank GEVD-MWF at mu = 1 is the MWF (Q diag(l / (l + 1)) Q^-1 e_0 = (Rss + Rnn)^-1 Rss e_0)
        other = "r1-mwf" if (typ, rank, mu) == ("gevd", "full", 1.0) else {"gevd": "mwf", "mwf": "gevd",
                                                                          "r1-mwf": "mwf"}[typ]
        out.append(("type", other, 1, mu, ref))
    return out


def _check_values(case, got, truth, port_fn, names, K, what):
    """Per (node, output): complex rel-L2 against float64 within TOL, else the fallback of record_parity against the
    fp32 port.  Records complex and magnitude rows.  Returns the bar the case was held to."""
    bar = TOL
    port = None
    for nm in names:
        for k in range(K):
            g, t = got[nm][k], truth[nm][k]
            assert np.isfinite(g.real).all() and np.isfinite(g.imag).all(), (what, nm, k, "not finite")
            e, em = rel_l2(g, t), rel_l2_mag(g, t)
            er = pe = erm = pem = None
            if e >= TOL:
                if port is None:
                    port = port_fn()
                er, pe = rel_l2(g, port[nm][k]), rel_l2(port[nm][k], t)
                erm, pem = rel_l2_mag(g, port[nm][k]), rel_l2_mag(port[nm][k], t)
                bar = max(bar, 1.25 * pe + 1e-6)
            ok = record_parity(case, nm, k, err_ref=er, err_f64=e, ref_f64=pe,
                               note="complex rel-L2; reference = fp32 port (oracle/tango_np)")
            assert ok, (what, nm, k, "complex", e, er, pe)
            # recorded next to it for comparison with the magnitude metric's rows; the case is judged on the complex one
            record_parity(case, nm + "|mag", k, err_ref=erm, err_f64=em, ref_f64=pem,
                          note="magnitude rel-L2 (recorded; the case is judged on the complex row)")
    return bar


def _hann(N):
    return 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(N) / N)


def _frame_env(x, n_fft):
    """[..., L] -> [..., T] sum_n w_n |xpad[t H + n]| (the STFT bound's envelope, DESIGN §2)."""
    H = n_fft // 2
    pad = np.pad(np.abs(np.asarray(x, np.float64)), [(0, 0)] * (x.ndim - 1) + [(H, H)], mode="reflect")
    T = 1 + x.shape[-1] // H
    idx = np.arange(n_fft)[None, :] + H * np.arange(T)[:, None]
    return pad[..., idx] @ _hann(n_fft)


def _check_zn(Yr, z, zn, extra=None, what=""):
    """zn = Yr - z entry-wise to one rounding (plus `extra`, a bound on the error of Yr)."""
    Yr, z, zn = (np.asarray(a).astype(np.complex128) for a in (Yr, z, zn))
    err = np.abs(zn - (Yr - z))
    bound = 2 * U * (np.abs(Yr) + np.abs(z)) + (0 if extra is None else extra)
    bad = ~(err <= bound)
    assert not bad.any(), "%s: zn != Y[ref] - z_y at %d entries, worst ratio %.3g" % (
        what, int(bad.sum()), float(np.max(err / np.maximum(bound, 1e-300))))


def _filter_env(args, B, K):
    """sum_d |w_d| |x_d| [B, K, T, F] of a filter_sum call's arguments (x = own channels, then z of the other nodes)."""
    W, Y, Z = args["W"], args["Y"], args["Z"]
    C = Y.shape[2]
    env = torch.einsum("bkfc,bkctf->bktf", W[..., :C].abs(), Y.abs())
    if Z is not None and K > 1:
        for k in range(K):
            others = [j for j in range(K) if j != k]
            env[:, k] += torch.einsum("bfj,bjtf->btf", W[:, k, :, C:].abs(), Z[:, others].abs())
    return env


# ---- offline routes ---------------------------------------------------------------------------------------------------
def _make_inputs(row, fi):
    from disco_b200.synth import make_batch, make_utterance
    K, C, n_fft = row["K"], row["C"], row["n_fft"]
    L = case_length(row)
    seed = 5000 + 100 * ROUTES.index(row) + fi
    if row["chans"] is not None:
        per = [make_utterance(seed + 10 * k, 1, c, L) for k, c in enumerate(row["chans"])]
        return [[p[i][0] for p in per] for i in range(3)], L
    y, s, n = make_batch(row["B"], K, C, L, seed0=seed)
    return (y, s, n), L


def _external(rng, B, K, T, F):
    return rng.uniform(0.05, 0.95, size=(B, K, T, F)).astype(np.float32)


def _estimator(mw, seen):
    """A step-2 mask estimator as tango_batched calls it: records what it is given and returns the mask mw (a fixed
    stand-in for a network's output; a mask computed from z_y and zn would make step 2 ill-conditioned here)."""
    def est(Y, z_y, zn):
        seen.append((Y, z_y.clone(), zn.clone()))
        return mw
    return est


@pytest.mark.parametrize("fi", range(len(FILTERS)), ids=["%s-r%s-mu%g" % f for f in FILTERS])
@pytest.mark.parametrize("row", ROUTES, ids=[r["id"] for r in ROUTES])
def test_route(dev, monkeypatch, row, fi):
    if row["chans"] is not None:
        return _ragged_case(dev, monkeypatch, row, fi)
    from disco_b200 import ops
    from disco_b200.tango import tango_batched
    typ, rank, mu, ref, kind, layout = case_options(row, fi)
    K, C, n_fft, B, mfz, vads = row["K"], row["C"], row["n_fft"], row["B"], row["mfz"], row["vads"]
    (y, s, n), L = _make_inputs(row, fi)
    T, F = ops.n_frames(L, n_fft), n_fft // 2 + 1
    case = "route_%s_%s_r%s_mu%g_ref%d_%s_%s" % (row["id"], typ, rank, mu, ref, kind, layout)
    yd, sd, nd = (torch.from_numpy(a).to(dev) for a in (y, s, n))
    rng = np.random.default_rng(17 * fi + ROUTES.index(row))
    mz_ext = mw_ext = None
    seen = []
    if kind == "external" or (kind == "callable" and fi % 2) or kind == "same":
        mz_ext = torch.from_numpy(_external(rng, B, K, T, F)).to(dev)
    if kind in ("external", "callable"):
        mw_ext = torch.from_numpy(_external(rng, B, K, T, F)).to(dev)

    def run(out_layout, diagnostics):
        if kind == "oracle":
            masks = None
        elif kind == "callable":
            if mz_ext is None:
                S, N = ops.stft(sd, n_fft), ops.stft(nd, n_fft)
                mz = ops.tf_mask(S[:, :, ref].contiguous(), N[:, :, ref].contiguous(), vads[0])
            else:
                mz = mz_ext
            masks = (mz, _estimator(mw_ext, seen))
        else:
            masks = (mz_ext, mw_ext)
        return tango_batched(yd, sd, nd, masks=masks, vads=vads, mask_for_z=mfz, n_fft=n_fft, mu=mu,
                             filter_type=typ, rank=rank, ref_mic=ref, out_layout=out_layout, diagnostics=diagnostics)

    spy = Spy(monkeypatch)
    out = run(layout, True)
    torch.cuda.synchronize()
    what = case
    # 1. spy
    hit = spy.sites()
    assert set(row["calls"]) <= hit, (what, "missing", sorted(set(row["calls"]) - hit))
    assert not (set(row["never"]) & hit), (what, "unexpected", sorted(set(row["never"]) & hit))
    spy.check_options(typ, rank, mu, ref, what)
    rec = list(spy.calls)
    # the outputs in [B, K, T, F]
    tf = (lambda a: a) if layout == "TF" else (lambda a: a.transpose(-1, -2))
    o = {k: tf(v) for k, v in out.items()}
    # 2. masks
    S, N = ops.stft(sd, n_fft), ops.stft(nd, n_fft)
    if kind == "oracle":
        want = ops.tf_mask(S[:, :, ref].contiguous(), N[:, :, ref].contiguous(), vads[0])
        assert torch.equal(o["masks_z"], want), (what, "masks_z is not the mask of microphone ref_mic")
        if vads[1] == vads[0] and ref == 0:
            assert out["mask_w"] is out["masks_z"], (what, "mask_w should reuse mask_z")
        else:
            want_w = ops.tf_mask(S[:, :, 0].contiguous(), N[:, :, 0].contiguous(), vads[1])
            assert torch.equal(o["mask_w"], want_w), (what, "mask_w is not the mask of microphone 0")
    elif kind in ("external", "same"):
        assert torch.equal(o["masks_z"], mz_ext), what
        assert torch.equal(o["mask_w"], mz_ext if kind == "same" else mw_ext), what
    else:
        assert len(seen) == 1 and torch.equal(o["mask_w"], mw_ext), what
        Yr, zr, znr = seen[0]
        y_site = [a for a in rec if a[0] in ("tango_step1:stft_scm#1", "tango_step1:stft_scm#2", "tango_step1:stft")]
        Yroute = y_site[0][3] if y_site[0][1] == "stft" else y_site[0][3][0]
        assert torch.equal(Yr, Yroute.view(Yr.shape)), (what, "the estimator did not get the route's Y")
        assert torch.equal(zr, o["z_y"]) and torch.equal(znr, o["zn"]), (what, "estimator inputs")
        if mz_ext is not None:
            assert torch.equal(o["masks_z"], mz_ext), what
    # 4. zn = Y[ref] - z_y with the route's Y
    Yrec = [a for a in rec if a[0] in ("tango_step1:stft_scm#1", "tango_step1:stft_scm#2", "tango_step1:stft")]
    zy, zn = o["z_y"].cpu().numpy(), o["zn"].cpu().numpy()
    if Yrec:
        Yroute = Yrec[0][3] if Yrec[0][1] == "stft" else Yrec[0][3][0]
        Yroute = Yroute.view(B, K, C, T, F)
        _check_zn(Yroute[:, :, ref].cpu().numpy(), zy, zn, what=what)
    else:
        Ys = ops.stft(yd.view(B * K, C, L), n_fft).view(B, K, C, T, F)[:, :, ref].cpu().numpy()
        tol_fft = math.sqrt(2) * (4 * math.log2(n_fft) + 6) * U
        E = _frame_env(y, n_fft)                                      # [B, K, C, T]
        extra = 2 * tol_fft * (E[:, :, ref] + E.max(axis=2))[..., None]
        _check_zn(Ys, zy, zn, extra, what + " (fuse_dual against ops.stft)")
    # 5. invariances: the other layout, and no diagnostics
    other = "TF" if layout == "FT" else "FT"
    spy.clear()
    out2 = run(other, True)
    rec2 = list(spy.calls)
    o2 = {k: (v if other == "TF" else v.transpose(-1, -2)) for k, v in out2.items()}
    assert set(out2) == set(out), what
    for nm in out:
        if nm in ("yf", "sf", "nf") and K > 1:
            # TF runs filter_sum_multi, FT the per-node filter_sum: both within the filter bound of float64
            tf_rec = rec if layout == "TF" else rec2
            call = [a for a in tf_rec if a[1] == "filter_sum" and a[3] is (out if layout == "TF" else out2)[nm]]
            assert call, (what, nm, "no filter_sum produced it")
            env = _filter_env(call[0][2], B, K)
            D = C + K - 1
            err = (o[nm] - o2[nm]).abs()
            assert bool((err <= 2 * 2 * math.sqrt(2) * (D + 1) * U * env).all()), (what, nm, "FT vs TF beyond bound")
        else:
            assert torch.equal(o[nm], o2[nm]), (what, nm, "FT output is not the transposed TF output")
    spy.clear()
    out3 = run(layout, False)
    for nm in ("yf", "z_y", "zn"):
        assert torch.equal(out3[nm], out[nm]), (what, nm, "diagnostics changed it")
    # 3. values against float64, per utterance and node
    names = ("yf", "sf", "nf", "z_y", "z_s", "z_n", "zn")
    Dmax = C + K - 1
    for b in range(B):
        got = {nm: _ft(o[nm][b]) for nm in names}
        if kind == "oracle":
            masks = None
        else:
            masks = (_ft(o["masks_z"][b]), _ft(o["mask_w"][b]))        # float32, as the kernels saw them
        orc = lambda t=typ, r=rank, m=mu, rf=ref, mk=masks, dp=True: f64_oracle(
            row, y[b], s[b], n[b], mk, vads, rf, t, r, m, mfz, double_port=dp)
        truth = orc()
        port_fn = lambda: orc(dp=False)
        bar = _check_values(case + "_b%d" % b, got, truth, port_fn, names, K, what)
        # 6. discrimination
        far = lambda a, nm: max(rel_l2(a[nm][k], truth[nm][k]) for k in range(K))
        for label, t2, r2, m2, rf2 in _neighbours(typ, rank, mu, ref, C, Dmax):
            alt = orc(t=t2, r=r2, m=m2, rf=rf2)
            d = max(far(alt, nm) for nm in names)
            assert d > 10 * bar, (what, "neighbour %s is only %.3g from the oracle (bar %.3g)" % (label, d, bar))
        for nm, fake in (("yf", np.conj(got["yf"])), ("zn", -got["zn"])):
            assert max(rel_l2(fake[k], truth[nm][k]) for k in range(K)) > 10 * bar, (what, "checker accepts", nm)
        if masks is not None and not np.array_equal(masks[0], masks[1]):
            sw = orc(mk=(masks[1], masks[0]))
            assert far(sw, "yf") > 10 * bar or far(sw, "z_y") > 10 * bar, (what, "checker accepts swapped masks")
        elif kind == "oracle" and not (vads[0] == vads[1] and ref == 0):
            mz, mw = _oracle_masks_f64(s[b], n[b], vads, ref, n_fft)
            sw = orc(mk=(mw, mz))
            assert far(sw, "yf") > 10 * bar or far(sw, "z_y") > 10 * bar, (what, "checker accepts swapped masks")


def _ragged_case(dev, monkeypatch, row, fi):
    """offline_tango on nodes of [2, 3, 2] microphones (reference microphone 0): spy, masks, values against
    tango_np(double=True), zn, discrimination.  The adapter has one layout and always computes the diagnostics."""
    from disco_b200 import ops
    from disco_b200.tango import offline_tango
    typ, rank, mu, _, kind, _ = case_options(row, fi)
    ref, mfz, vads, n_fft = 0, row["mfz"], row["vads"], row["n_fft"]
    (y, s, n), L = _make_inputs(row, fi)
    K = len(y)
    T, F = ops.n_frames(L, n_fft), n_fft // 2 + 1
    case = "route_%s_%s_r%s_mu%g_%s" % (row["id"], typ, rank, mu, kind)
    masks = None
    if kind == "external":
        rng = np.random.default_rng(31 + fi)
        masks = tuple([rng.uniform(0.05, 0.95, size=(F, T)).astype(np.float32) for _ in range(K)] for _ in range(2))
    spy = Spy(monkeypatch)
    res = offline_tango(y, s, n, list(vads), [None, None], mfz, n_fft=n_fft, mu=mu, filter_type=typ, rank=rank,
                        masks=masks)
    hit = spy.sites()
    assert set(row["calls"]) <= hit, (case, "missing", sorted(set(row["calls"]) - hit))
    assert not (set(row["never"]) & hit), (case, "unexpected", sorted(set(row["never"]) & hit))
    spy.check_options(typ, rank, mu, ref, case)
    names9 = ("yf", "sf", "nf", "z_y", "z_s", "z_n", "zn", "masks_z", "mask_w")
    got = {nm: [np.asarray(a) for a in v] for nm, v in zip(names9, res)}
    # masks: microphone 0 of each channel-count group's own STFT, or the external ones unchanged
    groups = {}
    for k in range(K):
        groups.setdefault(len(y[k]), []).append(k)
    Ys = [a for a in spy.calls if a[0] in ("tango_step1:stft_scm#1", "tango_step1:stft_scm#2", "tango_step1:stft")]
    assert len(Ys) == len(groups), case
    for (C, nodes), Yc in zip(sorted(groups.items()), Ys):
        sg = torch.from_numpy(np.stack([np.stack(s[k]) for k in nodes])[None]).to(dev)
        ng = torch.from_numpy(np.stack([np.stack(n[k]) for k in nodes])[None]).to(dev)
        S, N = ops.stft(sg, n_fft), ops.stft(ng, n_fft)
        for i, k in enumerate(nodes):
            if kind == "oracle":
                mz = ops.tf_mask(S[:, :, 0].contiguous(), N[:, :, 0].contiguous(), vads[0])[0, i]
                assert np.array_equal(got["masks_z"][k], _ft(mz)), (case, k)
            else:
                assert np.array_equal(got["masks_z"][k], masks[0][k]) and np.array_equal(got["mask_w"][k],
                                                                                           masks[1][k]), (case, k)
            Yroute = Yc[3] if Yc[1] == "stft" else Yc[3][0]
            Yroute = Yroute.view(1, len(nodes), C, T, F)
            _check_zn(Yroute[0, i, ref].cpu().numpy().T, got["z_y"][k], got["zn"][k], what="%s node %d" % (case, k))
    names = ("yf", "sf", "nf", "z_y", "z_s", "z_n", "zn")
    mk = None if masks is None else (np.array(masks[0]), np.array(masks[1]))
    orc = lambda t=typ, r=rank, m=mu, dp=True, mks=mk: f64_oracle(row, y, s, n, mks, vads, 0, t, r, m, mfz,
                                                                 double_port=dp)
    truth = orc()
    bar = _check_values(case, {nm: got[nm] for nm in names}, truth, lambda: orc(dp=False), names, K, case)
    far = lambda a, nm: max(rel_l2(a[nm][k], truth[nm][k]) for k in range(K))
    for label, t2, r2, m2, _ in _neighbours(typ, rank, mu, 0, 1, 2):     # C = 1: no other reference microphone
        alt = orc(t=t2, r=r2, m=m2)
        d = max(far(alt, nm) for nm in names)
        assert d > 10 * bar, (case, "neighbour %s is only %.3g from the oracle" % (label, d))
    for nm, fake in (("yf", [np.conj(a) for a in got["yf"]]), ("zn", [-a for a in got["zn"]])):
        assert max(rel_l2(fake[k], truth[nm][k]) for k in range(K)) > 10 * bar, (case, "checker accepts", nm)
    if mk is not None:
        sw = orc(mks=(mk[1], mk[0]))
        assert far(sw, "yf") > 10 * bar, (case, "checker accepts swapped masks")


# ---- online_tango -------------------------------------------------------------------------------------------------------
def _oracle_online(Y, mz, mw, lam, block, lag, fsel, ref, rank, R0):
    """oracle/online_np.online_mwf with the float64 solver per utterance and node on the bins fsel, Y [B, K, C, F, T]
    complex128 (float64 STFT), masks [B, K, T, F]; R0 (Rs0, Rn0) [B, K, F, C, C] or None seeds step 1, and step 2 too
    when K = 1.  -> z_y, zn, yf [B, K, len(fsel), T]."""
    from oracle import online_np, solve_f64, tango_np
    B, K, C = Y.shape[:3]
    fn = (tango_np.spatial_correlation_matrix, lambda Rs, Rn, mu, ft, r: solve_f64.solve(Rs, Rn, mu, ft, r))
    kw = dict(lambda_cor=lam, block=block, lag=lag, rank=rank, ref=ref)
    r0 = lambda b, k: None if R0 is None else (R0[0][b, k][fsel], R0[1][b, k][fsel])
    Ys = Y[:, :, :, fsel]
    z1 = np.stack([np.stack([online_np.online_mwf(Ys[b, k], mz[b, k].T[fsel], *fn, R0=r0(b, k), **kw)[0]
                             for k in range(K)]) for b in range(B)])
    zn = Ys[:, :, ref] - z1
    yf = np.empty_like(z1)
    for b in range(B):
        for k in range(K):
            X = Ys[b, k] if K == 1 else np.concatenate([Ys[b, k], z1[b, [j for j in range(K) if j != k]]], axis=0)
            yf[b, k] = online_np.online_mwf(X, mw[b, k].T[fsel], *fn, R0=r0(b, k) if K == 1 else None, **kw)[0]
    return z1, zn, yf


def _prior(Y64, mz, n=20):
    """(Rs0, Rn0) [B, K, F, C, C] complex64 of the scale of the data: the masked SCMs of the first n frames of Y64
    [B, K, C, F, T] under mz [B, K, T, F], exactly Hermitian with real diagonals."""
    C = Y64.shape[2]
    m = mz.transpose(0, 1, 3, 2)[:, :, None, :, :n]
    out = []
    for w in (m, 1 - m):
        X = w * Y64[..., :n]
        R = (np.einsum("bkcft,bkdft->bkfcd", X, X.conj()) / n).astype(np.complex64)
        R = 0.5 * (R + R.conj().swapaxes(-1, -2))
        R.imag[..., np.arange(C), np.arange(C)] = 0
        out.append(np.ascontiguousarray(R))
    return out


@pytest.mark.parametrize("row", ONLINE, ids=[r["id"] for r in ONLINE])
def test_online_tango_options(dev, monkeypatch, row):
    """online_tango at non-default ref_mic, rank, lag, block and R0 against the float64 composition: complex values
    from block ceil(4 D / block) + lag on within 1e-5, finite everywhere; frames before the first filter equal Y[ref]
    exactly in z_y and yf; each neighbouring option moves the oracle more than 10x the bar."""
    from disco_b200 import online, ops
    from disco_b200.synth import make_batch
    from oracle import librosa_np
    K, C, n_fft, block, lag, rank = row["K"], row["C"], row["n_fft"], row["block"], row["lag"], row["rank"]
    ref = C - 1 if row["ref"] == "last" else 0
    B, L, lam = 2, 24000, 0.98
    y, s, n = make_batch(B, K, C, L, seed0=7000 + 10 * ONLINE.index(row))
    S, N = (ops.stft(torch.from_numpy(a[:, :, 0]).contiguous().to(dev), n_fft) for a in (s, n))
    mz, mw = ops.tf_mask(S, N, "irm1"), ops.tf_mask(S, N, "irm2")
    T, F = mz.shape[-2:]
    Y64 = np.stack([np.stack([np.stack([librosa_np.stft(y[b, k, c].astype(np.float64), n_fft=n_fft,
                                                        hop_length=n_fft // 2) for c in range(C)])
                              for k in range(K)]) for b in range(B)])          # [B, K, C, F, T]
    prior = _prior(Y64, mz.cpu().numpy())
    R0 = prior if row["R0"] else None
    spy = Spy(monkeypatch)
    r0d = None if R0 is None else tuple(torch.from_numpy(r).to(dev) for r in R0)
    on = online.online_tango(torch.from_numpy(y).to(dev), (mz, mw), lambda_cor=lam, block=block, lag=lag, rank=rank,
                             ref_mic=ref, n_fft=n_fft, R0=r0d)
    torch.cuda.synchronize()
    what = "online %s ref=%d rank=%d lag=%d block=%d R0=%s n_fft=%d" % (row["id"], ref, rank, lag, block, row["R0"],
                                                                       n_fft)
    assert set(row["calls"]) <= spy.sites(), (what, sorted(set(row["calls"]) - spy.sites()))
    spy.check_options("gevd", rank, 1.0, ref, what)
    rec = [a for a in spy.calls if a[1] == "scm_recursive"]
    assert len(rec) == 2, what
    for i, (_, _, args, _) in enumerate(rec):
        want_r0 = R0 is not None and (i == 0 or K == 1)
        assert (args["R0"] is not None) == want_r0, (what, "step %d R0" % (i + 1))
        if want_r0:
            assert all(a is b for a, b in zip(args["R0"], r0d)), what
    Yd = [a for a in spy.calls if a[0] == "online_tango:stft"][0][3]
    for key in ("yf", "z_y", "zn"):
        assert on[key].shape == (B, K, T, F) and bool(torch.isfinite(torch.view_as_real(on[key])).all()), (what, key)
    # pass-through frames: channel ref of Y, exactly, in z_y and yf
    t_first = min(T, lag * block)
    if lag >= 1:
        for key in ("z_y", "yf"):
            assert torch.equal(on[key][:, :, :t_first], Yd[:, :, ref, :t_first]), (what, key, "pass-through frames")
    fsel = [0, 37, F // 2, F - 1]
    z1, zn1, yf1 = _oracle_online(Y64, mz.cpu().numpy(), mw.cpu().numpy(), lam, block, lag, fsel, ref, rank, R0)
    got = {k: on[k].cpu().numpy()[:, :, :, fsel].transpose(0, 1, 3, 2) for k in ("z_y", "zn", "yf")}
    truth = {"z_y": z1, "zn": zn1, "yf": yf1}
    start = {k: (-(-4 * D // block) + lag) * block for k, D in (("z_y", C), ("zn", C), ("yf", C + K - 1))}
    assert max(start.values()) < T - block, what
    for k in truth:
        e = rel_l2(got[k][..., start[k]:], truth[k][..., start[k]:])
        assert e <= TOL, "%s: %s from frame %d: complex rel %.3g" % (what, k, start[k], e)
    # discrimination
    alts = [("ref_mic", dict(ref=C - 1 if ref == 0 else 0)), ("rank", dict(rank=2 if rank == 1 else 1)),
            ("lag", dict(lag={0: 1, 1: 0, 2: 1}[lag])), ("R0", dict(R0=None if R0 is not None else "prior"))]
    for label, ch in alts:
        a = dict(ref=ref, rank=rank, lag=lag, R0=R0)
        a.update(ch)
        if a["R0"] == "prior":
            a["R0"] = prior
        oz, ozn, oyf = _oracle_online(Y64, mz.cpu().numpy(), mw.cpu().numpy(), lam, block, a["lag"], fsel, a["ref"],
                                      a["rank"], a["R0"])
        alt = {"z_y": oz, "zn": ozn, "yf": oyf}
        d = max(rel_l2(alt[k][..., start[k]:], truth[k][..., start[k]:]) for k in truth)
        assert d > 10 * TOL, (what, "neighbour %s is only %.3g from the oracle" % (label, d))
