"""Every instantiation of the step-2 and online kernels against float64, at the frame counts where its tiling has
edges, at all three STFT sizes, through the C ABI with every output inside a NaN-filled guard band.

Dispatch targets and what selects them (INSTANCES below lists the instantiations; tests/test_kernel_instances_cpu.py
parses the dispatch sets out of the sources and requires this table to cover exactly them):
  masked_scm        scm.cu       masked_scm_kernel<D, ZF, FC>, D = C + K - 1 <= 4; ZF = fused z (filter_sum_scm),
                                 FC = 257 at n_fft 512, runtime F otherwise
  masked_scm_wide   scm_wide.cu  masked_scm_wide_kernel, D 5..16 (NPART 1 / 2 / 4), ZF for D 5..8 (K = 1)
  tango_mid         mid_multi.cu tango_mid_kernel<C, K, ...>, the (C, K) of tango_mid_supported
  filter_sum        filter_sum.cu  filter_sum_tf_kernel<D, FC> (frame-major out), filter_sum_kernel<D> ((F, T) out)
  filter_sum_multi  filter_sum_multi.cu  filter_sum_multi_kernel<C, K>: K > 1, all nodes, frame-major out, Z [B, K]
  online            online.cu    scm_blocks_kernel<D> + scm_combine_kernel, filter_sum_blocks_kernel<D>

Tolerances are entry-wise and scaled by absolute values, so that no bin, frame or matrix entry can hide in a norm.
Float32 summation of n terms in a fixed order, each term formed with a few roundings, errs by at most
(n + roundings per term) * u * sum |term| per real component (u = 2^-24, first order), so at most sqrt(2) times that
in modulus:
  SCMs     |R_ij - R_ij^f64| <= tol * (1/T) sum_t w_t |x_i| |x_j|, with
           tol = sqrt(2) * (ceil(T / ways) + (ways - 1) + 5 + 6) * u: each of the `ways` time-ways sums its frames
           sequentially, the ways are added in fixed order (ways - 1), the Nyquist block closes with a 5-level lane
           butterfly, and 6 covers the roundings of one term (m^2, the two of the complex product, the fma into the
           accumulator) and of the 1/T scale (1/T itself and the product).
  filters  |out - out^f64| <= tol * sum_d |w_d| |x_d|, tol = 2 sqrt(2) * (D + 1) * u: D complex fmas, each two
           roundings per component; the residual x_ref - out adds one rounding of at most u |x_ref| + u |out|.
  online   the block sum has P terms and the combine walks J blocks, each an fma with a rounded lambda^P:
           tol = sqrt(2) * (P + J + 6) * u against the envelope lambda^(t+1) |R0| + sum (1 - lambda) lambda^(t - s) w_s |x_i||x_j|.
These are bounds, not fits: rounding errors add up to far less on random data, while a dropped frame, a wrong stride
or a wrong pair index is an O(1) error.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
SENTINEL = 0x7FC0DEAD     # a quiet-NaN bit pattern no kernel computes
GUARD = 1024              # 32-bit words (4 KB) of sentinel before and after every output; keeps 16-byte alignment
N_FFTS = (256, 512, 1024)  # F = 129, 257 (the FC = 257 instantiations), 513

MID_PAIRS = ((1, 2), (2, 2), (3, 2), (4, 2), (1, 3), (2, 3), (3, 3), (4, 3), (1, 4), (2, 4), (3, 4), (4, 4),
             (2, 8), (4, 8), (2, 6))
# one row per dispatch target: the instantiations its launcher selects from
INSTANCES = {
    "masked_scm": {"D": (1, 2, 3, 4), "zf_D": (1, 2, 3, 4)},
    "masked_scm_wide": {"D": tuple(range(5, 17)), "zf_D": (5, 6, 7, 8)},
    "tango_mid": {"CK": MID_PAIRS},
    "filter_sum": {"D": tuple(range(1, 17))},
    "filter_sum_multi": {"CK": MID_PAIRS},
    "online": {"D": tuple(range(1, 9))},
}


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


# ---- tiling of each kernel, read off its source -----------------------------------------------------------------

def scm_geom(D):
    """(time-ways, frames per tile): scm.cu ScmGeom has TW = 8 ways of one frame each per round; scm_wide.cu
    launch_wide_dz has NPART = 1 / 2 / 4 pair partitions, TW = 8 / NPART ways, TS = 8 (TW >= 4) or 4 frames a tile."""
    if D <= 4:
        return 8, 8
    tw = 8 // (1 if D <= 6 else (2 if D <= 8 else 4))
    return tw, (8 if tw >= 4 else 4)


def edge_frames(ts, extra=()):
    """T = 1; just below, at and above one tile; just below and above 32 tiles (one tile of the Nyquist block, whose
    lanes walk frames); a long ragged sequence."""
    return sorted({1, max(1, ts - 1), ts, ts + 1, 32 * ts - 1, 32 * ts + 1, 301, *extra})


MID_TS = 4     # mid_multi.cu MidCfg::TS and filter_sum_multi.cu FsmCfg::TS
FILTER_TS = 8  # filter_sum.cu: 8 warps = time-ways; 2 x UF frames per way and round, UF = 2 for D <= 4; (F, T)
               # output in tiles of 32 frames


def tol_scm(T, ways):
    return math.sqrt(2) * (math.ceil(T / ways) + (ways - 1) + 5 + 6) * U


def tol_filter(D):
    return 2 * math.sqrt(2) * (D + 1) * U


# ---- outputs inside sentinel-filled guard bands -----------------------------------------------------------------

class Guarded:
    """Output tensors carved out of larger buffers filled with a NaN bit pattern.  check() asserts that the kernels
    wrote every word of every output and not one word of the guard bands around them."""

    def __init__(self, dev):
        self.dev, self.bufs = dev, []

    def new(self, shape):
        n = 2 * int(np.prod(shape))                       # complex64 = two 32-bit words
        buf = torch.full((n + 2 * GUARD,), SENTINEL, dtype=torch.int32, device=self.dev)
        self.bufs.append((buf, n))
        return buf[GUARD:GUARD + n].view(torch.complex64).view(shape)

    def check(self, what):
        torch.cuda.synchronize()
        for i, (buf, n) in enumerate(self.bufs):
            assert bool((buf[:GUARD] == SENTINEL).all()), "%s: output %d: write before its start" % (what, i)
            assert bool((buf[GUARD + n:] == SENTINEL).all()), "%s: output %d: write past its end" % (what, i)
            left = int((buf[GUARD:GUARD + n] == SENTINEL).sum())
            assert left == 0, "%s: output %d: %d of %d words never written" % (what, i, left, n)
        self.bufs = []


def _sel_arg(sel):
    if sel is None:
        return None, 0
    return (ctypes.c_int * len(sel))(*sel), len(sel)


def _call(fn, *args):
    from disco_b200 import _lib, ops
    _lib.check(getattr(_lib.load(), fn)(*args, ops._stream()))


def _p(t):
    from disco_b200 import ops
    return ops._ptr(t)


# ---- inputs and float64 references ------------------------------------------------------------------------------

def cplx(rng, *s):
    return (rng.standard_normal(s) + 1j * rng.standard_normal(s)).astype(np.complex64)


class Step2:
    """Step-2 input of B utterances of K nodes: own spectra Y [n_grp, C, T, F] of the selected nodes and the
    compressed signals Z [B, K, T, F] of all nodes; group g = (utterance g // n_sel, node sel[g % n_sel])."""

    def __init__(self, rng, dev, B, C, K, T, F, sel=None, z_layout="BK", mask="TF"):
        self.B, self.C, self.K, self.T, self.F, self.sel = B, C, K, T, F, sel
        self.nodes = list(range(K)) if sel is None else list(sel)
        self.n_grp = B * len(self.nodes)
        self.D = C + K - 1
        self.Y = cplx(rng, self.n_grp, C, T, F)
        self.Z = cplx(rng, B, K, T, F) if K > 1 else None
        self.m = rng.uniform(size=(self.n_grp, T, F)).astype(np.float32) if mask else None
        self.mask_layout = mask
        self.z_layout = z_layout
        self.Yd = torch.from_numpy(self.Y).to(dev)
        self.Zd = None
        if K > 1:
            Zh = self.Z if z_layout == "BK" else np.ascontiguousarray(self.Z.transpose(1, 0, 2, 3))
            self.Zd = torch.from_numpy(Zh).to(dev)
        self.md = None
        if mask:
            mh = self.m if mask == "TF" else np.ascontiguousarray(self.m.transpose(0, 2, 1))
            self.md = torch.from_numpy(mh).to(dev)

    @property
    def lay(self):
        return 1 if self.mask_layout == "FT" else 0

    @property
    def zl(self):
        return 1 if self.z_layout == "KB" else 0

    @property
    def n_utt(self):
        return self.B if self.K > 1 else self.n_grp

    def X(self, g):
        """[own mics ; z of the other nodes in node order] of group g, (D, T, F) complex64."""
        if self.K == 1:
            return self.Y[g]
        b, k = divmod(g, len(self.nodes))
        k = self.nodes[k]
        return np.concatenate([self.Y[g], self.Z[b, [j for j in range(self.K) if j != k]]], axis=0)

    def groups(self):
        return [(self.X(g), None if self.m is None else self.m[g]) for g in range(self.n_grp)]


def ref_scm(X, m):
    """X (D, T, F), m (T, F) or None -> Rss, Rnn (F, D, D) complex128 and their envelopes (1/T) sum_t w |x_i||x_j|."""
    D, T, F = X.shape
    Xf = np.ascontiguousarray(X.astype(np.complex128).transpose(2, 0, 1))       # (F, D, T)
    A = np.abs(Xf)
    if m is None:
        wa, wb = np.ones((F, T)), np.zeros((F, T))
    else:
        m = m.astype(np.float64).T
        wa, wb = m * m, (1 - m) * (1 - m)
    XH, AT = Xf.conj().transpose(0, 2, 1), A.transpose(0, 2, 1)
    R = np.concatenate([Xf * wa[:, None], Xf * wb[:, None]], axis=1) @ XH / T
    E = np.concatenate([A * wa[:, None], A * wb[:, None]], axis=1) @ AT / T
    return R[:, :D], R[:, D:], E[:, :D], E[:, D:]


def assert_bounded(got, want, env, tol, what):
    err = np.abs(got.astype(np.complex128) - want)
    bad = ~(err <= tol * env)                                 # NaN counts as out of bound
    if bad.any():
        idx = tuple(np.argwhere(bad)[0])
        raise AssertionError("%s: %d of %d entries out of bound; first at %s: |err| %.3g, bound %.3g (tol %.3g)"
                             % (what, int(bad.sum()), bad.size, idx, err[idx], tol * env[idx], tol))


def check_scm(Rss, Rnn, groups, tol, what):
    """Every (group, bin, i, j) against float64, groups = [(X, mask)]; exact Hermitian mirrors and real diagonals;
    Rnn = 0 without a mask."""
    for R in (Rss, Rnn):
        assert torch.equal(R, R.conj().transpose(-1, -2)), what + ": mirrors not exactly conjugate"
        assert not bool(torch.diagonal(torch.view_as_real(R), dim1=-3, dim2=-2)[..., 1, :].any()), \
            what + ": diagonal with an imaginary part"
    Rs, Rn = Rss.cpu().numpy(), Rnn.cpu().numpy()
    for g, (X, m) in enumerate(groups):
        if m is None:
            assert not np.any(Rn[g]), what + ": Rnn not exactly 0 without a mask"
        ws, wn, es, en = ref_scm(X, m)
        assert_bounded(Rs[g], ws, es, tol, "%s Rss group %d" % (what, g))
        assert_bounded(Rn[g], wn, en, tol, "%s Rnn group %d" % (what, g))


def ref_filter(W, X, conj):
    """W (F, D), X (D, T, F) -> out (T, F) complex128 and the envelope sum_d |w_d||x_d|."""
    W = W.astype(np.complex128)
    out = np.einsum("fd,dtf->tf", W.conj() if conj else W, X.astype(np.complex128))
    env = np.einsum("fd,dtf->tf", np.abs(W), np.abs(X).astype(np.float64))
    return out, env


def check_filter(out, resid, W, X, conj, ref, what):
    """out, resid (T, F) numpy against float64, entry-wise."""
    want, env = ref_filter(W, X, conj)
    tol = tol_filter(X.shape[0])
    assert_bounded(out, want, env, tol, what + " out")
    if resid is not None:
        xr = X[ref].astype(np.complex128)
        assert_bounded(resid, xr - want, env + np.abs(xr) + np.abs(want), tol, what + " resid")


# ---- masked_scm / masked_scm_wide -------------------------------------------------------------------------------

def splits(D):
    """(C, K) with C + K - 1 = D: one node, two, four and D single-microphone nodes, as far as they exist."""
    out = [(D, 1)]
    for K in (2, 4, D):
        if 2 <= K <= D and (D - K + 1, K) not in out:
            out.append((D - K + 1, K))
    return out


def node_subset(K, i):
    """All nodes, or a proper subset (the ragged-array launch) that includes the last node."""
    if K == 1 or i % 2 == 0:
        return None
    return [K - 1] if K == 2 else [0, K - 1]


def run_masked_scm(dev, prob, n_fft):
    o = Guarded(dev)
    shape = (prob.n_grp, prob.F, prob.D, prob.D)
    Rss, Rnn = o.new(shape), o.new(shape)
    sel, n_sel = _sel_arg(prob.sel)
    _call("disco_masked_scm", _p(prob.Yd), _p(prob.Zd), _p(prob.md), prob.lay, _p(Rss), _p(Rnn), prob.n_utt, prob.K,
          prob.C, prob.T, n_fft, sel, n_sel, prob.zl)
    o.check("masked_scm")
    return Rss, Rnn


SCM_DS = INSTANCES["masked_scm"]["D"] + INSTANCES["masked_scm_wide"]["D"]


@pytest.mark.parametrize("n_fft", N_FFTS)
@pytest.mark.parametrize("D", SCM_DS)
def test_masked_scm_every_instance(dev, D, n_fft):
    """masked_scm at D = C + K - 1 over one node, several nodes (utterance- and node-major Z, node subsets), masks in
    (T, F), in (F, T) and none, at every tile edge of the kernel that D selects."""
    ways, ts = scm_geom(D)
    F = n_fft // 2 + 1
    sp = splits(D)
    for i, T in enumerate(edge_frames(ts, extra=(2 * ts + 1, 4 * ts + 1))):
        rng = np.random.default_rng(1000 * D + T + n_fft)
        C, K = sp[i % len(sp)]
        mask = ("TF", "FT", None)[i % 3]
        prob = Step2(rng, dev, 2 if K <= 4 and T < 64 else 1, C, K, T, F, sel=node_subset(K, i),
                     z_layout="KB" if (i // 2) % 2 else "BK", mask=mask)
        Rss, Rnn = run_masked_scm(dev, prob, n_fft)
        check_scm(Rss, Rnn, prob.groups(), tol_scm(T, ways), "D=%d C=%d K=%d T=%d mask=%s" % (D, C, K, T, mask))


@pytest.mark.parametrize("n_fft", N_FFTS)
@pytest.mark.parametrize("C", INSTANCES["masked_scm"]["zf_D"] + INSTANCES["masked_scm_wide"]["zf_D"])
def test_filter_sum_scm_every_instance(dev, C, n_fft):
    """The fused step-1 filter + SCM (K = 1, D = C): z and zn against float64, and matrices bit-identical to those of
    masked_scm on the same input."""
    ways, ts = scm_geom(C)
    F = n_fft // 2 + 1
    for i, T in enumerate(edge_frames(ts, extra=(2 * ts + 1, 4 * ts + 1))):
        rng = np.random.default_rng(2000 * C + T + n_fft)
        prob = Step2(rng, dev, 2 if T < 64 else 1, C, 1, T, F, mask=("TF", "FT")[i % 2])
        ref = (C - 1, 0, C // 2)[i % 3]
        W1 = cplx(rng, prob.n_grp, F, C)
        o = Guarded(dev)
        z, zn = o.new((prob.n_grp, T, F)), o.new((prob.n_grp, T, F))
        Rss, Rnn = o.new((prob.n_grp, F, C, C)), o.new((prob.n_grp, F, C, C))
        _call("disco_filter_sum_scm", _p(torch.from_numpy(W1).to(dev)), _p(prob.Yd), _p(prob.md), prob.lay, _p(z),
              _p(zn), ref, _p(Rss), _p(Rnn), prob.n_grp, C, T, n_fft)
        what = "C=%d T=%d" % (C, T)
        o.check("filter_sum_scm " + what)
        Rss2, Rnn2 = run_masked_scm(dev, prob, n_fft)
        assert torch.equal(Rss, Rss2) and torch.equal(Rnn, Rnn2), what
        check_scm(Rss, Rnn, prob.groups(), tol_scm(T, ways), what)
        zh, znh = z.cpu().numpy(), zn.cpu().numpy()
        for g in range(prob.n_grp):
            check_filter(zh[g], znh[g], W1[g], prob.Y[g], True, ref, "%s group %d z" % (what, g))


# ---- tango_mid --------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n_fft", N_FFTS)
@pytest.mark.parametrize("C,K", INSTANCES["tango_mid"]["CK"])
def test_tango_mid_every_instance(dev, C, K, n_fft):
    """The fused multi-node middle pass: z, zn against float64, the SCMs against float64 of [Y_k ; z_j] (the z it
    wrote), and equal to filter_sum + masked_scm to the tolerances of test_gpu_parity."""
    from conftest import rel_l2
    from disco_b200 import ops
    F, D = n_fft // 2 + 1, C + K - 1
    for i, T in enumerate(edge_frames(MID_TS, extra=(4 * MID_TS + 1,))):
        rng = np.random.default_rng(3000 * C + 100 * K + T + n_fft)
        B = 2 if T < 64 else 1
        ref = (C - 1, 0)[i % 2]
        Y, W1 = cplx(rng, B * K, C, T, F), cplx(rng, B * K, F, C)
        m = rng.uniform(size=(B * K, T, F)).astype(np.float32)
        Yd, Wd, md = (torch.from_numpy(a).to(dev) for a in (Y, W1, m))
        o = Guarded(dev)
        z, zn = o.new((B, K, T, F)), o.new((B, K, T, F))
        Rss, Rnn = o.new((B * K, F, D, D)), o.new((B * K, F, D, D))
        _call("disco_tango_mid", _p(Wd), _p(Yd), _p(md), _p(z), _p(zn), ref, _p(Rss), _p(Rnn), B, K, C, T, n_fft)
        what = "C=%d K=%d T=%d" % (C, K, T)
        o.check("tango_mid " + what)
        zh, znh = z.cpu().numpy().reshape(B * K, T, F), zn.cpu().numpy().reshape(B * K, T, F)
        for g in range(B * K):
            check_filter(zh[g], znh[g], W1[g], Y[g], True, ref, "%s group %d z" % (what, g))
        zb = zh.reshape(B, K, T, F)
        groups = [(np.concatenate([Y[b * K + k], zb[b, [j for j in range(K) if j != k]]]), m[b * K + k])
                  for b in range(B) for k in range(K)]
        check_scm(Rss, Rnn, groups, tol_scm(T, 1), what)
        z2, zn2 = ops.filter_sum(Wd.view(B, K, F, C), Yd.view(B, K, C, T, F), None, conj=True, ref=ref, n_fft=n_fft)
        Rss2, Rnn2 = ops.masked_scm(Yd.view(B, K, C, T, F), md.view(B, K, T, F), z2, n_fft=n_fft)
        assert rel_l2(z.cpu().numpy(), z2.cpu().numpy()) < 1e-6 and rel_l2(zn.cpu().numpy(), zn2.cpu().numpy()) < 1e-6
        assert rel_l2(Rss.cpu().numpy(), Rss2.view(B * K, F, D, D).cpu().numpy()) < 2e-6, what
        assert rel_l2(Rnn.cpu().numpy(), Rnn2.view(B * K, F, D, D).cpu().numpy()) < 2e-6, what


# ---- filter_sum (per-node kernels) and filter_sum_multi ---------------------------------------------------------

def run_filter_sum(dev, prob, W, conj, ref, out_ft):
    o = Guarded(dev)
    shape = (prob.n_grp, prob.F, prob.T) if out_ft else (prob.n_grp, prob.T, prob.F)
    out, resid = o.new(shape), o.new(shape)
    sel, n_sel = _sel_arg(prob.sel)
    _call("disco_filter_sum", _p(torch.from_numpy(W).to(dev)), int(conj), _p(prob.Yd), _p(prob.Zd), _p(out),
          _p(resid), ref, int(out_ft), prob.n_utt, prob.K, prob.C, prob.T, 2 * (prob.F - 1), sel, n_sel, prob.zl)
    o.check("filter_sum")
    out, resid = out.cpu().numpy(), resid.cpu().numpy()
    if out_ft:
        out, resid = out.transpose(0, 2, 1), resid.transpose(0, 2, 1)
    return out, resid


def check_filter_sum(prob, W, out, resid, conj, ref, what):
    for g in range(prob.n_grp):
        check_filter(out[g], resid[g], W[g], prob.X(g), conj, ref, "%s group %d" % (what, g))


@pytest.mark.parametrize("n_fft", N_FFTS)
@pytest.mark.parametrize("D", INSTANCES["filter_sum"]["D"])
def test_filter_sum_every_instance(dev, D, n_fft):
    """The per-node filter-and-sum, frame-major and (F, T) output, conj and plain taps, the residual against a
    microphone and against a compressed channel, node subsets and node-major Z (K > 1 with all nodes, frame-major
    output and utterance-major Z goes to filter_sum_multi instead, tested below)."""
    F = n_fft // 2 + 1
    sp = splits(D)
    T_list = sorted({1, FILTER_TS - 1, FILTER_TS, FILTER_TS + 1, 2 * FILTER_TS + 1, 31, 32, 33, 255, 257, 301})
    for i, T in enumerate(T_list):
        rng = np.random.default_rng(4000 * D + T + n_fft)
        C, K = sp[i % len(sp)]
        out_ft = i % 2 == 1
        sel, zl = None, "BK"
        if K > 1 and not out_ft:
            sel, zl = ([K - 1] if K == 2 else [0, K - 1], "BK") if i % 4 == 0 else (None, "KB")
        elif K > 1:
            sel = node_subset(K, i // 2)
        prob = Step2(rng, dev, 2 if K <= 4 and T < 64 else 1, C, K, T, F, sel=sel, z_layout=zl, mask=None)
        conj = i % 3 != 2
        ref = (D - 1) if (K > 1 and i % 2 == 0) else (i % C)
        W = cplx(rng, prob.n_grp, F, D)
        out, resid = run_filter_sum(dev, prob, W, conj, ref, out_ft)
        check_filter_sum(prob, W, out, resid, conj, ref, "D=%d C=%d K=%d T=%d ft=%d" % (D, C, K, T, out_ft))


@pytest.mark.parametrize("n_fft", N_FFTS)
@pytest.mark.parametrize("C,K", INSTANCES["filter_sum_multi"]["CK"])
def test_filter_sum_multi_every_instance(dev, C, K, n_fft):
    """The all-nodes filter-and-sum.  Its launcher splits the frame tiles of an (utterance, bin block) over gridDim.z
    up to (T / 4 + 7) / 8 segments, so many utterances of under 32 frames run with gridDim.z = 1 and one utterance of
    127 or more frames with several segments (some of them empty in the Nyquist block, whose tiles span 128 frames)."""
    F, D = n_fft // 2 + 1, C + K - 1
    for i, T in enumerate(edge_frames(MID_TS, extra=(4 * MID_TS + 1,))):
        rng = np.random.default_rng(5000 * C + 100 * K + T + n_fft)
        prob = Step2(rng, dev, 12 if T < 32 else 1, C, K, T, F, mask=None)
        conj = i % 2 == 0
        ref = (C - 1, D - 1, C)[i % 3]
        W = cplx(rng, prob.n_grp, F, D)
        out, resid = run_filter_sum(dev, prob, W, conj, ref, False)
        check_filter_sum(prob, W, out, resid, conj, ref, "C=%d K=%d T=%d" % (C, K, T))


# ---- online ------------------------------------------------------------------------------------------------------

# (T, block, lag, power, R0, mask): block 1, blocks that do not divide T, block 64 (the largest), lags 0 / 1 / 2
ONLINE_CASES = [(1, 1, 0, 2, False, True), (3, 5, 1, 1, True, False), (64, 64, 0, 2, True, True),
                (151, 5, 2, 1, False, True), (151, 1, 1, 2, True, True), (151, 64, 1, 1, True, False),
                (129, 7, 0, 2, False, False)]


def check_recursive(Rss, Rnn, X, m, lam, P, power, R0, tol, what):
    """Per-frame complex128 recursion R <- lam R + (1 - lam) w x x^H, with the same recursion on absolute values as the
    envelope, compared with the kernel's matrices after every block of P frames.  All groups at once: Rss, Rnn
    (G, J, F, D, D) from the kernel, X (G, D, T, F), m (G, T, F) or None, R0 (Rs0, Rn0) (G, F, D, D) or None."""
    G, D, T, F = X.shape
    X = X.astype(np.complex128)
    if R0 is None:
        R = [np.zeros((G, F, D, D), np.complex128) for _ in range(2)]
    else:
        R = [r.astype(np.complex128) for r in R0]
    E = [np.abs(r) for r in R]
    for t in range(T):
        x = X[:, :, t].transpose(0, 2, 1)                      # (G, F, D)
        xx = x[..., :, None] * x[..., None, :].conj()
        aa = np.abs(x)[..., :, None] * np.abs(x)[..., None, :]
        if m is None:
            w = (np.ones((G, F)), np.zeros((G, F)))
        else:
            mt = m[:, t].astype(np.float64)
            w = (mt * mt, (1 - mt) ** 2) if power == 2 else (mt, 1 - mt)
        for s in range(2):
            R[s] = lam * R[s] + (1 - lam) * w[s][..., None, None] * xx
            E[s] = lam * E[s] + (1 - lam) * w[s][..., None, None] * aa
        if (t + 1) % P == 0 or t == T - 1:
            j = t // P
            assert_bounded(Rss[:, j], R[0], E[0], tol, "%s Rss block %d" % (what, j))
            assert_bounded(Rnn[:, j], R[1], E[1], tol, "%s Rnn block %d" % (what, j))


@pytest.mark.parametrize("n_fft", N_FFTS)
@pytest.mark.parametrize("D", INSTANCES["online"]["D"])
def test_online_every_instance(dev, D, n_fft):
    """scm_recursive (block sums + combine) against the per-frame float64 recursion at every block end, and
    filter_sum_blocks against float64 with its pass-through before the first filter exact."""
    F = n_fft // 2 + 1
    sp = splits(D)
    lam = 0.93
    for i, (T, P, lag, power, with_r0, with_mask) in enumerate(ONLINE_CASES):
        rng = np.random.default_rng(6000 * D + 10 * i + n_fft)
        C, K = sp[i % len(sp)]
        prob = Step2(rng, dev, 2 if K <= 4 and T < 64 else 1, C, K, T, F, sel=node_subset(K, i),
                     mask="TF" if with_mask else None)
        J = (T + P - 1) // P
        R0 = None
        if with_r0:
            R0 = []
            for _ in range(2):       # exactly Hermitian, as the recursion keeps it
                a = cplx(rng, prob.n_grp, F, D, D).astype(np.complex128)
                r = np.triu((a @ a.conj().transpose(0, 1, 3, 2) / D).astype(np.complex64))
                r = r + np.triu(r, 1).conj().transpose(0, 1, 3, 2)
                r.imag[..., np.arange(D), np.arange(D)] = 0
                R0.append(r)
        what = "D=%d C=%d K=%d T=%d block=%d power=%d R0=%d mask=%d" % (D, C, K, T, P, power, with_r0, with_mask)
        o = Guarded(dev)
        Rss, Rnn = o.new((prob.n_grp, J, F, D, D)), o.new((prob.n_grp, J, F, D, D))
        r0d = [torch.from_numpy(r).to(dev) for r in R0] if with_r0 else [None, None]
        sel, n_sel = _sel_arg(prob.sel)
        _call("disco_scm_recursive", _p(prob.Yd), _p(prob.Zd), _p(prob.md), _p(r0d[0]), _p(r0d[1]), _p(Rss), _p(Rnn),
              ctypes.c_double(lam), P, power, prob.n_utt, K, C, T, n_fft, sel, n_sel)
        o.check("scm_recursive " + what)
        assert torch.equal(Rss, Rss.conj().transpose(-1, -2)) and torch.equal(Rnn, Rnn.conj().transpose(-1, -2))
        Rs, Rn = Rss.cpu().numpy(), Rnn.cpu().numpy()
        if not with_mask and not with_r0:
            assert not np.any(Rn), what + ": Rnn not exactly 0 without a mask"
        check_recursive(Rs, Rn, np.stack([prob.X(g) for g in range(prob.n_grp)]), prob.m, lam, P, power, R0,
                        math.sqrt(2) * (P + J + 6) * U, what)

        conj = i % 2 == 0
        ref = (D - 1) if (K > 1 and i % 3 == 0) else (i % C)
        W = cplx(rng, prob.n_grp, J, F, D)
        o = Guarded(dev)
        out, resid = o.new((prob.n_grp, T, F)), o.new((prob.n_grp, T, F))
        _call("disco_filter_sum_blocks", _p(torch.from_numpy(W).to(dev)), int(conj), _p(prob.Yd), _p(prob.Zd),
              _p(out), _p(resid), ref, P, lag, prob.n_utt, K, C, T, n_fft, sel, n_sel)
        o.check("filter_sum_blocks " + what)
        out, resid = out.cpu().numpy(), resid.cpu().numpy()
        t_first = min(T, lag * P)                              # frames before the first filter pass channel `ref`
        for g in range(prob.n_grp):
            X = prob.X(g)
            assert np.array_equal(out[g, :t_first], X[ref, :t_first]), what
            assert not np.any(resid[g, :t_first]), what
            for j in range(lag, J):
                t0, t1 = j * P, min(T, (j + 1) * P)
                check_filter(out[g, t0:t1], resid[g, t0:t1], W[g, j - lag], X[:, t0:t1], conj, ref,
                             "%s lag=%d group %d block %d" % (what, lag, g, j))
