"""TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

Frame-by-frame float64 restatement of the recursive MWF step whose speech and noise statistics read their own channel
stacks: the step-1 statistics of online Tango's 'use_oracle_*' exchange modes (the scans of S and N) and the step 2 of
every mode other than 'local' ([mask_w Y_own ; z_rs] and [(1 - mask_w) Y_own ; z_rn]), as disco_b200/online.py
evaluates them.  Like oracle/online_np.online_mwf it composes the reference's spatial_correlation_matrix (M=None, every
frame) and intern_filter (every block), injected as `scm` and `solve`.  Xs = m X, Xn = (1 - m) X gives
online_np.online_mwf(X, m, power=2).
"""
import numpy as np


def online_mwf_split(X, Xs, Xn, scm, solve, lambda_cor=0.95, block=8, lag=1, mu=1.0, filter_type="gevd", rank=1,
                     ref=0, R0=None):
    """Every frame updates R_ss with the frame of Xs and R_nn with that of Xn; the filter of every block applies to X.
    X, Xs, Xn (D, F, T) complex; R0 = (R0ss, R0nn) (F, D, D) or None.  Returns z (F, T), W (J, F, D), Rss, Rnn
    (J, F, D, D) -- the smoothed matrices after the last frame of every block."""
    D, F, T = X.shape
    J = (T + block - 1) // block
    Rss = np.zeros((F, D, D), dtype=np.complex128) if R0 is None else np.array(R0[0], dtype=np.complex128)
    Rnn = np.zeros((F, D, D), dtype=np.complex128) if R0 is None else np.array(R0[1], dtype=np.complex128)
    snap_s = np.zeros((J, F, D, D), dtype=np.complex128)
    snap_n = np.zeros_like(snap_s)
    W = np.zeros((J, F, D), dtype=np.complex128)
    z = np.zeros((F, T), dtype=np.complex128)
    for t in range(T):
        j = t // block
        for f in range(F):
            Rss[f] = scm(Rss[f], Xs[:, f, t].astype(np.complex128), lambda_cor)
            Rnn[f] = scm(Rnn[f], Xn[:, f, t].astype(np.complex128), lambda_cor)
            jw = j - lag
            w = W[jw, f] if jw >= 0 else np.eye(D)[ref]
            z[f, t] = np.inner(np.conj(w), X[:, f, t].astype(np.complex128))
        if t == min(T, (j + 1) * block) - 1:      # block complete: refresh the filter
            snap_s[j], snap_n[j] = Rss, Rnn
            for f in range(F):
                W[j, f] = solve(Rss[f], Rnn[f], mu, filter_type, rank)[0]
            if lag == 0:                          # look-ahead variant: re-filter the block with its own filter
                for tt in range(j * block, t + 1):
                    z[:, tt] = np.einsum("fd,df->f", np.conj(W[j]), X[:, :, tt])
    return z, W, snap_s, snap_n
