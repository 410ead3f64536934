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

A batch of utterances of different lengths runs in one call (`online_tango(..., lengths=)`, `online_mwf(...,
frames=)`): every utterance's outputs are those of the utterance run alone, in the batch's T_max shapes and exactly
0 past its own frames and blocks.
"""
import torch

from . import ops
from .tango import _frame_clip, _uneven_lengths


def online_mwf(Y, mask, Z=None, lambda_cor=0.95, block=8, lag=1, mu=1.0, filter_type="gevd", rank=1, ref=0, power=2,
               R0=None, n_fft=512, frames=None):
    """One recursive MWF step.  Y [B, K, C, T, F] complex64, mask [B, K, T, F] float32, Z [B, K, T, F] compressed
    signals of all nodes (step 2) or None (step 1).  Returns dict(z, zn [B, K, T, F]; W [B, K, J, F, D]; Rss, Rnn).
    frames: None, or host integers, one per utterance in [1, T]: utterance b is its first frames[b] frames (nothing
    later is read); z, zn are 0 from frame frames[b] on, Rss, Rnn and W from block ceil(frames[b] / block) on."""
    Rss, Rnn = ops.scm_recursive(Y, mask, Z, lambda_cor, block, power, R0, n_fft, frames=frames)
    W, _ = ops.mwf_solve(Rss, Rnn, mu, filter_type, rank)
    if frames is not None:   # the solver saw the zero matrices past each utterance's blocks: drop what it made of them
        J = W.shape[2]
        n_blk = -(-torch.from_numpy(ops.signal_lengths(frames, Y.shape[:1], Y.shape[3]).astype("int64")) // block)
        live = torch.arange(J) < n_blk[:, None]
        W = torch.where(live.to(W.device)[:, None, :, None, None], W, torch.zeros((), dtype=W.dtype, device=W.device))
    z, zn = ops.filter_sum_blocks(W, Y, Z, block, lag, True, ref, n_fft, frames=frames)
    return {"z": z, "zn": zn, "W": W, "Rss": Rss, "Rnn": Rnn}


def _uneven_batch(y, masks, lens, n_fft):
    """The spectra of an uneven batch (stft_lengths: 0 past each utterance's frames), its per-utterance frame counts
    and the masks set to 0 past them (a selection: a NaN there stays out of the statistics)."""
    Y = ops.stft_lengths(y, lens, n_fft)
    clip = _frame_clip(lens, Y.shape[3], n_fft, Y.device)
    return Y, ops.n_frames(lens, n_fft), [clip(m) for m in masks]


def online_tango(y, masks, lambda_cor=0.95, block=8, lag=1, mu=1.0, rank=1, ref_mic=0, n_fft=512, R0=None,
                 lengths=None):
    """Two-step recursive Tango on time signals y [B, K, C, L]: local recursive MWF -> exchange of the compressed
    signals z -> recursive MWF on [own mics ; z of the other nodes] (the channel order of concatenate_signals,
    tango.py:142-155).  masks = (mask_z, mask_w) [B, K, T, F] frame-major; R0 = optional initial (R_ss, R_nn) of the
    local step [B, K, F, C, C] (the second step of a multi-node array starts from zeros).  Returns yf, z_y, zn
    [B, K, T, F] and the per-block filters W1, W2.

    lengths: None, or one length in samples per utterance, n_fft / 2 < lengths[b] <= L (as tango_batched takes
    them).  Utterance b is then y[b, ..., :lengths[b]] with T_b = 1 + lengths[b] // hop frames: its yf, z_y, zn are
    those of the utterance run alone on frames t < T_b and 0 from T_b on, its W1, W2 those of the lone run on blocks
    j < ceil(T_b / block) and 0 after; masks past T_b are ignored.  Bit-identical to the lone run when K * C is even
    (the STFT transforms signals 2p, 2p + 1 together; DESIGN §5).  post.to_time(yf, L, lengths=lengths) turns the
    outputs into signals per utterance."""
    mask_z, mask_w = masks
    mask_w = mask_z if mask_w is None else mask_w
    lens = _uneven_lengths(lengths, y.shape[0], y.shape[-1], n_fft)   # None: the uniform batch
    frames = None
    if lens is None:
        Y = ops.stft(y, n_fft)
    else:
        Y, frames, (mask_z, mask_w) = _uneven_batch(y, (mask_z, mask_w), lens, n_fft)
    s1 = online_mwf(Y, mask_z, None, lambda_cor, block, lag, mu, "gevd", rank, ref_mic, 2, R0, n_fft, frames)
    K = Y.shape[1]
    if K == 1:
        s2 = online_mwf(Y, mask_w, None, lambda_cor, block, lag, mu, "gevd", rank, ref_mic, 2, R0, n_fft, frames)
    else:
        s2 = online_mwf(Y, mask_w, s1["z"].contiguous(), lambda_cor, block, lag, mu, "gevd", rank, ref_mic, 2, None,
                        n_fft, frames)
    return {"yf": s2["z"], "z_y": s1["z"], "zn": s1["zn"], "W1": s1["W"], "W2": s2["W"]}
