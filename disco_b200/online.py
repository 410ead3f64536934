"""Online (recursive) variant of the MWF steps (SURVEY.md §8 f-4).

The reference ships one streaming primitive, `spatial_correlation_matrix(Rxx, x, lambda_cor, M)`
(se_utils/internal_formulas.py:84-103: R <- lambda R + (1 - lambda) [M] x x^H for ONE frame and bin), next to
the batch filter `intern_filter`.  Composed per frame they give the causal counterpart of an `offline_tango`
step: exponentially smoothed masked SCMs, a filter refreshed every `block` frames from the statistics seen
so far, applied to the following frames.  Here that composition is three batched launches over all
utterances, nodes, bins and blocks (csrc/online.cu + the batched solver):

    scm_recursive      scan of the recursion -> (R_ss, R_nn) after every block; D = C + K - 1 <= 8: two levels
                       (block sums, then the combine), 9..16: one staged pass that carries R (same values)
    mwf_solve          one GEVD-MWF per (block, bin)
    filter_sum_blocks  frame t filtered with the filter of block t // block - lag

Every channel stack up to D = 16 runs, the MEETIT geometry (8 nodes x 2 mics, step 2 at D = 9) included;
the chunked `stream.OnlineTangoStream` covers D <= 8.

`lag = 1` is strictly causal with an algorithmic delay of 0 frames (the filter in force was finished before
the frame arrived); `lag = 0` uses the block's own statistics (look-ahead of up to block - 1 frames).
"""
import torch

from . import ops


def online_mwf(Y, mask, Z=None, lambda_cor=0.95, block=8, lag=1, mu=1.0, filter_type="gevd", rank=1, ref=0, power=2,
               R0=None, n_fft=512):
    """One recursive MWF step.  Y [B, K, C, T, F] complex64, mask [B, K, T, F] float32, Z [B, K, T, F] compressed
    signals of all nodes (step 2) or None (step 1).  Returns dict(z, zn [B, K, T, F]; W [B, K, J, F, D]; Rss, Rnn)."""
    Rss, Rnn = ops.scm_recursive(Y, mask, Z, lambda_cor, block, power, R0, n_fft)
    W, _ = ops.mwf_solve(Rss, Rnn, mu, filter_type, rank)
    z, zn = ops.filter_sum_blocks(W, Y, Z, block, lag, True, ref, n_fft)
    return {"z": z, "zn": zn, "W": W, "Rss": Rss, "Rnn": Rnn}


def online_tango(y, masks, lambda_cor=0.95, block=8, lag=1, mu=1.0, rank=1, ref_mic=0, n_fft=512, R0=None):
    """Two-step recursive Tango on time signals y [B, K, C, L]: local recursive MWF -> exchange of the compressed
    signals z -> recursive MWF on [own mics ; z of the other nodes] (the channel order of concatenate_signals,
    tango.py:142-155).  masks = (mask_z, mask_w) [B, K, T, F] frame-major; R0 = optional initial (R_ss, R_nn) of the
    local step [B, K, F, C, C] (the second step of a multi-node array starts from zeros).  Returns yf, z_y, zn
    [B, K, T, F] and the per-block filters W1, W2."""
    mask_z, mask_w = masks
    mask_w = mask_z if mask_w is None else mask_w
    Y = ops.stft(y, n_fft)
    s1 = online_mwf(Y, mask_z, None, lambda_cor, block, lag, mu, "gevd", rank, ref_mic, 2, R0, n_fft)
    K = Y.shape[1]
    if K == 1:
        s2 = online_mwf(Y, mask_w, None, lambda_cor, block, lag, mu, "gevd", rank, ref_mic, 2, R0, n_fft)
    else:
        s2 = online_mwf(Y, mask_w, s1["z"].contiguous(), lambda_cor, block, lag, mu, "gevd", rank, ref_mic, 2, None,
                        n_fft)
    return {"yf": s2["z"], "z_y": s1["z"], "zn": s1["zn"], "W1": s1["W"], "W2": s2["W"]}
