"""One kernel, a few launches, nothing else from this library: the target of `ncu --set full`.

    ncu --set full --clock-control none --import-source on -k regex:<kernel> -s 2 -c 1 -o out python scripts/prof_target.py <what>

what: stft_scm2 | stft_scm2_noY | stft_filter_dual | stft_filter_dual_ft | stft_scm1 | stft | stft_scm_c8 | stft_scm_c8_256 | filter_dual | masked_scm_zf4 | filter_sum4 | istft |
      solve4 | solve8 | tango_mid44 | tango_mid28 | filter_multi44 | masked_scm_zf8
Shapes = the BASELINE workloads (64 x 4 mics x 10 s; 128 x 8 mics x 10 s; 64 x 4 nodes x 4 mics; 64 x 8 nodes x 2 mics)."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from disco_b200 import ops  # noqa: E402

what = sys.argv[1]
n = int(sys.argv[2]) if len(sys.argv) > 2 else 4
dev = torch.device("cuda:0")
g = torch.Generator().manual_seed(0)
L = 160000
cplx = lambda *s: torch.complex(torch.randn(s, generator=g), torch.randn(s, generator=g)).to(dev)
rnd = lambda *s: torch.rand(s, generator=g).to(dev)


def TF(n_fft):
    return 1 + L // (n_fft // 2), n_fft // 2 + 1


if what in ("stft_scm2", "stft_scm2_noY", "stft_scm1", "stft", "stft_filter_dual", "stft_filter_dual_ft"):
    T, F = TF(512)
    x, m, m2 = torch.randn((64, 4, L), generator=g).to(dev), rnd(64, T, F), rnd(64, T, F)
    W1, W2 = cplx(64, F, 4), cplx(64, F, 4)
    fn = {"stft_scm2": lambda: ops.stft_scm2(x, m, m2), "stft_scm2_noY": lambda: ops.stft_scm2(x, m, m2, want_Y=False),
          "stft_scm1": lambda: ops.stft_scm(x, m, keep_partials=True), "stft": lambda: ops.stft(x),
          "stft_filter_dual": lambda: ops.stft_filter_dual(x, W1, W2),
          "stft_filter_dual_ft": lambda: ops.stft_filter_dual(x, W1, W2, out_layout="FT")}[what]
elif what in ("stft_scm_c8", "stft_scm_c8_256"):
    n_fft = 256 if what.endswith("256") else 512
    T, F = TF(n_fft)
    x, m = torch.randn((128, 8, L), generator=g).to(dev), rnd(128, T, F)
    fn = lambda: ops.stft_scm(x, m, n_fft, keep_partials=True)
elif what in ("filter_dual", "masked_scm_zf4", "filter_sum4", "solve4"):
    T, F = TF(512)
    Y, W1, W2, m = cplx(64, 1, 4, T, F), cplx(64, 1, F, 4), cplx(64, 1, F, 4), rnd(64, 1, T, F)
    if what == "solve4":
        x = torch.randn((64, 4, L), generator=g).to(dev)
        _, ws = ops.stft_scm2(x, m[:, 0].contiguous(), rnd(64, T, F))
        torch.cuda.synchronize()
        fn = lambda: ops.mwf_solve_workspace2(ws, 64, 4, L)
    else:
        fn = {"filter_dual": lambda: ops.filter_dual(W1, W2, Y), "masked_scm_zf4": lambda: ops.filter_sum_scm(W1, Y, m),
              "filter_sum4": lambda: ops.filter_sum(W1, Y, None)}[what]
elif what in ("masked_scm_zf8", "solve8"):
    T, F = TF(512)
    Y, W1, m = cplx(128, 1, 8, T, F), cplx(128, 1, F, 8), rnd(128, 1, T, F)
    if what == "solve8":
        Rss, Rnn = ops.masked_scm(Y, m, None)
        torch.cuda.synchronize()
        fn = lambda: ops.mwf_solve(Rss, Rnn)
    else:
        fn = lambda: ops.filter_sum_scm(W1, Y, m)
elif what in ("tango_mid44", "tango_mid28", "filter_multi44", "filter_multi28"):
    K, C = (4, 4) if what.endswith("44") else (8, 2)
    T, F = TF(512)
    D = C + K - 1
    Y, W1, m = cplx(64, K, C, T, F), cplx(64, K, F, C), rnd(64, K, T, F)
    if what.startswith("tango_mid"):
        fn = lambda: ops.tango_mid(W1, Y, m)
    else:
        Z, W2 = cplx(64, K, T, F), cplx(64, K, F, D)
        fn = lambda: ops.filter_sum(W2, Y, Z)
elif what == "istft":
    T, F = TF(512)
    Y = cplx(64, T, F)
    fn = lambda: ops.istft(Y, L)
else:
    raise SystemExit("unknown target " + what)

ops.init(512)
ops.init(256)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
for i in range(n):
    if i == n - 1:
        e0.record()
    fn()
e1.record()
torch.cuda.synchronize()
print("%s: last launch %.1f us" % (what, e0.elapsed_time(e1) * 1e3))
