"""Small end-to-end run for compute-sanitizer (memcheck / racecheck / synccheck)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from disco_b200 import ops
from disco_b200.synth import make_batch
from disco_b200.tango import tango_batched
dev = torch.device("cuda:0")
for (B, K, C, L, n_fft) in ((3, 2, 4, 9000, 512), (2, 1, 3, 5003, 256), (2, 3, 2, 6000, 1024)):
    y, s, n = make_batch(B, K, C, L, seed0=1)
    out = tango_batched(torch.from_numpy(y).to(dev), torch.from_numpy(s).to(dev), torch.from_numpy(n).to(dev), n_fft=n_fft)
    x = ops.istft(ops.stft(torch.from_numpy(y).to(dev), n_fft), L, n_fft)
    torch.cuda.synchronize()
    print("ok", B, K, C, L, n_fft, float(out["yf"].abs().mean()), float((x.cpu() - torch.from_numpy(y)).abs().max()))

# wide-channel engine (cp.async-staged), Nyquist block, fused z, ragged T; filter bank; online kernels
from disco_b200 import online, post
rng = np.random.default_rng(0)
cplx = lambda *s: torch.from_numpy((rng.standard_normal(s) + 1j * rng.standard_normal(s)).astype(np.complex64)).to(dev)
for (B, K, C, T, n_fft) in ((2, 1, 8, 37, 512), (2, 4, 4, 21, 256), (1, 8, 2, 9, 512), (2, 3, 13, 33, 256), (1, 2, 4, 300, 256)):
    F = n_fft // 2 + 1
    Y, W, Z = cplx(B, K, C, T, F), cplx(B, K, F, C), (cplx(B, K, T, F) if K > 1 else None)
    m = torch.rand(B, K, T, F, device=dev)
    Rs, Rn = ops.masked_scm(Y, m, Z, n_fft=n_fft)
    if K == 1:
        ops.filter_sum_scm(W, Y, m, ref=1, n_fft=n_fft)
    elif ops.tango_mid_supported(C, K):
        ops.tango_mid(W, Y, m, ref=0, n_fft=n_fft)
    o = online.online_mwf(Y, m, Z, block=4, lag=1, n_fft=n_fft)     # D 9..16: online_wide.cu
    if C + K - 1 > 8:   # the staged scan with R0, a block straddling its ring and a short last block
        Rs0 = torch.eye(C + K - 1, dtype=torch.complex64, device=dev).expand(B, K, F, C + K - 1, C + K - 1).contiguous()
        ops.scm_recursive(Y, m, Z, 0.9, 5, 2, (Rs0, Rs0.clone()), n_fft)
    torch.cuda.synchronize()
    print("ok wide", B, K, C, T, n_fft, float(Rs.abs().mean()))
# online Tango stream: streaming STFT / iSTFT with carried history, block buffers, a partial last block
from disco_b200.stream import OnlineTangoStream
for (B, K, C, n_fft, block, sizes) in ((3, 1, 3, 256, 4, (100, 0, 700, 1, 2500)), (2, 3, 2, 1024, 2, (513, 3000, 77))):
    s = OnlineTangoStream(B, K, C, n_fft=n_fft, block=block, lag=1, device=dev)
    fn = lambda t0, Y, z, zn: (torch.rand(z.shape, device=dev), None)
    for n in sizes:
        s.push(torch.randn(B, K, C, n, device=dev), fn)
    out = s.flush(fn)
    torch.cuda.synchronize()
    print("ok stream", B, K, C, n_fft, s.frames_out, s.samples_out, float(out["yf_time"].abs().mean()))
x = torch.randn(37, 3000, device=dev)
print("ok bank", float(post.fw_snr(x[:, 100:], 0.5 * torch.randn(37, 2900, device=dev), 16000)[1].mean()))
torch.cuda.synchronize()
# STOI: resampler, silent-frame selection (one all-silent clean), bands of cleans and pairs, a short pair (1e-5)
import warnings
from disco_b200 import stoi
x = torch.randn(3, 24000, device=dev) * (torch.arange(24000, device=dev) % 8000 < 5000)
x[1] = 0
with warnings.catch_warnings():
    warnings.simplefilter("ignore", RuntimeWarning)
    d = stoi.stoi_pairs(x, torch.cat((x + 0.3 * torch.randn_like(x), x[:, :5000].repeat(1, 5)[:, :24000])),
                        [(0, 0), (1, 1), (2, 2), (0, 3), (2, 5)], 16000)
    d_short = stoi.stoi(x[:, :3000], x[:, :3000], 16000)
torch.cuda.synchronize()
print("ok stoi", d.tolist(), d_short.tolist())
# signals of their own lengths: length-aware STFT / iSTFT at every n_fft (odd signal counts, pairs of equal and of
# different lengths, a signal of hop + 1 samples), the length-aware resampler and STOI selection, an uneven Tango batch
for n_fft in (256, 512, 1024):
    H = n_fft // 2
    L = 9 * H + 37
    lengths = [L, H + 1, L - H - 3, L - H - 3, 5 * H + 1]
    x = torch.randn(len(lengths), L, device=dev)
    for i, Lb in enumerate(lengths):
        x[i, Lb:] = 0
    Y = ops.stft_lengths(x, lengths, n_fft)
    xr = ops.istft_lengths(Y, lengths, L, n_fft)
    torch.cuda.synchronize()
    print("ok lengths", n_fft, float((xr - x).abs().max()))
with warnings.catch_warnings():
    warnings.simplefilter("ignore", RuntimeWarning)
    x = torch.randn(3, 24000, device=dev) * (torch.arange(24000, device=dev) % 8000 < 5000)
    d = stoi.stoi_pairs(x, x + 0.3 * torch.randn_like(x), [(0, 0), (1, 1), (2, 2)], 16000, lengths=[24000, 9001, 17777])
torch.cuda.synchronize()
y, s, n = make_batch(3, 2, 2, 9000, seed0=2)
out = tango_batched(torch.from_numpy(y).to(dev), torch.from_numpy(s).to(dev), torch.from_numpy(n).to(dev),
                    lengths=[9000, 5001, 7003])
td = post.to_time(out, 9000, lengths=[9000, 5001, 7003])
torch.cuda.synchronize()
print("ok lengths stoi / tango", d.tolist(), float(td["yf"].abs().mean()))
# online Tango on utterances of their own lengths: block edges, a one-block utterance, the staged wide scan (D = 9)
# with a block straddling its ring, R0, and filters / masks never read past each utterance's end
for (B, K, C, L, n_fft, block) in ((3, 1, 4, 6000, 512, 8), (3, 8, 2, 5000, 256, 5), (2, 1, 10, 4000, 1024, 1)):
    y, _, _ = make_batch(B, K, C, L, seed0=3)
    H = n_fft // 2
    lengths = [L, H + 1, 2 * block * H + 7][:B]
    T, F = 1 + L // H, H + 1
    masks = (torch.rand(B, K, T, F, device=dev), torch.rand(B, K, T, F, device=dev))
    R0 = None
    if K == 1:
        R0 = tuple(torch.eye(C, dtype=torch.complex64, device=dev).expand(B, K, F, C, C).contiguous() for _ in range(2))
    out = online.online_tango(torch.from_numpy(y).to(dev), masks, block=block, n_fft=n_fft, R0=R0, lengths=lengths)
    td = post.to_time(out, L, n_fft=n_fft, names=("yf", "z_y"), layout="TF", lengths=lengths)
    torch.cuda.synchronize()
    print("ok online lengths", B, K, C, n_fft, block, float(td["yf"].abs().mean()))
# pool of independent streams: per-slot STFT / iSTFT (odd K C: a lone last signal), slots opening, idling, closing and
# reopening, block closes on a subset of the slots
from disco_b200.stream import OnlineTangoPool
for (S, K, C, n_fft, block) in ((3, 1, 3, 256, 4), (2, 2, 3, 1024, 2), (2, 8, 2, 512, 3)):
    pool = OnlineTangoPool(S, K, C, n_fft=n_fft, block=block, device=dev)
    fn = lambda t0, n_fr, Y, z, zn: (torch.rand(z.shape, device=dev), None)
    H = n_fft // 2
    pool.open([0])
    pool.push(torch.randn(S, K, C, 3 * H + 5, device=dev), np.array([3 * H + 5] + [0] * (S - 1)), fn)
    pool.open(list(range(1, S)))
    for n in ((1, H - 1), (5 * H, 0), (0, 2 * H + 1)):
        nn = np.array([n[s % 2] for s in range(S)])
        pool.push(torch.randn(S, K, C, max(int(nn.max()), 1), device=dev), nn, fn)
    pool.close([0], fn)
    pool.open([0])
    pool.push(torch.randn(S, K, C, 4 * H, device=dev), np.full(S, 4 * H), fn)
    out = pool.close(list(range(S)), fn)
    torch.cuda.synchronize()
    print("ok pool", S, K, C, n_fft, pool.frames_out.tolist(), float(out["yf_time"].abs().mean()))
