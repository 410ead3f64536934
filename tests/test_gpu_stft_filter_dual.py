"""The fused STFT + dual filter (the filter pass of the single-node two-mask route) against the two-kernel sequence
it replaces, and the two-mask fused STFT+SCM without its spectrum against the run that stores it."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _cplx(rng, dev, *s):
    return torch.from_numpy((rng.standard_normal(s) + 1j * rng.standard_normal(s)).astype(np.complex64)).to(dev)


# (groups, samples): odd lengths put the reflect padding of both ends into partial edge tiles; 70 x 6000 and
# 200 x 1001 spread a few tiles per group over the persistent CTAs, so CTA ranges start and end inside groups and
# one CTA walks several groups; 3 x 64000 gives every CTA a run of tiles inside one group
SHAPES = [(3, 5003), (2, 4001), (70, 6000), (200, 1001), (3, 64000)]


@pytest.mark.parametrize("n_fft", [256, 512])
@pytest.mark.parametrize("C,refs", [(1, (0,)), (2, (0, 1)), (3, (0, 2)), (4, (1, 3))])
@pytest.mark.parametrize("layout", ["TF", "FT"])
def test_stft_filter_dual_equals_filter_dual_of_stft(dev, n_fft, C, refs, layout):
    """z, zn, yf bit-identical to filter_dual(W1, W2, stft(x)).  The reference spectrum is taken per group, so that a
    group's channels are paired in the two-for-one FFT exactly as in the fused kernel (odd C: the last channel alone)."""
    from disco_b200 import ops
    rng = np.random.default_rng(C * 7 + n_fft)
    F = n_fft // 2 + 1
    for G, L in SHAPES:
        x = torch.from_numpy(rng.standard_normal((G, C, L)).astype(np.float32)).to(dev)
        W1, W2 = _cplx(rng, dev, G, F, C), _cplx(rng, dev, G, F, C)
        Y = torch.stack([ops.stft(x[g], n_fft) for g in range(G)])
        for ref in refs:
            z, zn, yf = ops.stft_filter_dual(x, W1, W2, ref=ref, n_fft=n_fft, out_layout=layout)
            z0, zn0, yf0 = ops.filter_dual(W1, W2, Y, ref=ref, n_fft=n_fft, out_layout=layout)
            assert torch.equal(z, z0) and torch.equal(zn, zn0) and torch.equal(yf, yf0), (G, L, ref)
        z1, zn1, yf1 = ops.stft_filter_dual(x, W1, W2, ref=refs[-1], n_fft=n_fft, out_layout=layout, want_zn=False)
        assert zn1 is None and torch.equal(z1, z) and torch.equal(yf1, yf)


def test_stft_filter_dual_rejects_uncovered_shapes(dev):
    from disco_b200 import ops
    F = 257
    W = torch.zeros((1, F, 5), dtype=torch.complex64, device=dev)
    with pytest.raises(NotImplementedError):
        ops.stft_filter_dual(torch.zeros((1, 5, 4000), device=dev), W, W)
    W = torch.zeros((1, 513, 4), dtype=torch.complex64, device=dev)
    with pytest.raises(NotImplementedError):
        ops.stft_filter_dual(torch.zeros((1, 4, 4000), device=dev), W, W, n_fft=1024)


@pytest.mark.parametrize("n_fft", [256, 512])
@pytest.mark.parametrize("G,C,length", [(3, 4, 9000), (2, 3, 5003), (5, 1, 4000), (70, 4, 6000), (4, 2, 20000)])
@pytest.mark.parametrize("layout", ["TF", "FT"])
def test_stft_scm2_without_Y_same_workspace(dev, n_fft, G, C, length, layout):
    """The whole partial-sum workspace, slot for slot, with and without the spectrum store.  Both workspaces start
    from the same fill, so slots no CTA writes compare equal too."""
    from disco_b200 import _lib, ops
    rng = np.random.default_rng(G * 13 + C)
    x = torch.from_numpy(rng.standard_normal((G, C, length)).astype(np.float32)).to(dev)
    T, F = 1 + length // (n_fft // 2), n_fft // 2 + 1
    shape = (G, T, F) if layout == "TF" else (G, F, T)
    ma = torch.from_numpy(rng.uniform(size=shape).astype(np.float32)).to(dev)
    mb = torch.from_numpy(rng.uniform(size=shape).astype(np.float32)).to(dev)
    lib = _lib.load()
    nbytes = lib.disco_stft_scm2_workspace(G, C, length, n_fft)
    lay = ops._layout(layout)
    Y = torch.empty((G, C, T, F), dtype=torch.complex64, device=dev)
    stream = ops._stream()
    out = []
    for y in (Y, None):
        ws = torch.full((nbytes // 4,), -7.0, dtype=torch.float32, device=dev)
        _lib.check(lib.disco_stft_scm2(ops._ptr(x), ops._ptr(ma), ops._ptr(mb), lay, ops._ptr(y), G, C, length, n_fft,
                                       ops._ptr(ws), nbytes, stream))
        out.append(ws)
    assert torch.equal(out[0], out[1])
    assert torch.equal(Y, ops.stft_scm2(x, ma, mb, n_fft, mask_layout=layout)[0])
    Y0, ws0 = ops.stft_scm2(x, ma, mb, n_fft, mask_layout=layout, want_Y=False)
    assert Y0 is None and ws0.numel() == nbytes // 4
