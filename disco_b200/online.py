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

Every channel stack up to D = 16 runs, the MEETIT geometry (8 nodes x 2 mics, step 2 at D = 9) included, in
the whole-signal call and in the chunked `stream.OnlineTangoStream` alike (D >= 9 there with wide=True).

`lag = 1` is strictly causal with an algorithmic delay of 0 frames (the filter in force was finished before
the frame arrived); `lag = 0` uses the block's own statistics (look-ahead of up to block - 1 frames).

A batch of utterances of different lengths runs in one call (`online_tango(..., lengths=)`, `online_mwf(...,
frames=)`): every utterance's outputs are those of the utterance run alone, in the batch's T_max shapes and exactly
0 past its own frames and blocks.

Online Tango from clean components.  `online_tango(y, s=s, n=n, ...)` takes the evaluation inputs of
`tango.tango_batched` and returns its outputs, with the recursive steps in place of the batch ones:
    masks        masks=None builds them from s, n like tango_batched ('irmX' / 'ibmX' / 'iamX' / 'ivad' of
                 microphone ref_mic for step 1, of microphone 0 for step 2) and returns them as masks_z, mask_w;
                 a callable mask_w(Y, z_y, zn) is called after step 1
    mask_for_z   the exchange modes of tango._z_for_stats.  Other than 'local', step 2 takes R_ss as the unweighted
                 scan of [mask_w Y_own ; z_rs] and R_nn as that of [(1 - mask_w) Y_own ; z_rn] (tango_step2 with
                 z_rs / z_rn) and filters [Y_own ; z_y]; 'use_oracle_*' takes the step-1 statistics from the scans of
                 S and N.  With one node there is nothing to exchange: a non-'local' step 2 then differs from
                 'local' only by rounding, as (m y)(m y)^H is not rounded like m^2 y y^H
    diagnostics  z_s, z_n = W1 applied to S, N; sf, nf = W2 applied to [S_own ; z_s], [N_own ; z_n]; each one
                 filter_sum_blocks call with the block, lag, ref_mic and frames of yf, passing channel ref_mic
                 through before the first filter
so that post.to_time(out, L, n_fft, layout="TF", lengths=) and post.tango_scores score it like offline Tango.
"""
import torch

from . import ops
from .tango import _check_sources, _clean_masks, _frame_clip, _ref_plane, _uneven_lengths, _z_for_stats


def _live_blocks(W, frames, T, block):
    """W [B, K, J, F, D] with the blocks from ceil(frames[b] / block) on set to 0 (the solver saw the zero matrices
    past each utterance's blocks: drop what it made of them); W itself for frames=None."""
    if frames is None:
        return W
    J = W.shape[2]
    n_blk = -(-torch.from_numpy(ops.signal_lengths(frames, W.shape[:1], T).astype("int64")) // block)
    live = torch.arange(J) < n_blk[:, None]
    return torch.where(live.to(W.device)[:, None, :, None, None], W, torch.zeros((), dtype=W.dtype, device=W.device))


def online_mwf(Y, mask, Z=None, lambda_cor=0.95, block=8, lag=1, mu=1.0, filter_type="gevd", rank=1, ref=0, power=2,
               R0=None, n_fft=512, frames=None):
    """One recursive MWF step.  Y [B, K, C, T, F] complex64, mask [B, K, T, F] float32, Z [B, K, T, F] compressed
    signals of all nodes (step 2) or None (step 1).  Returns dict(z, zn [B, K, T, F]; W [B, K, J, F, D]; Rss, Rnn).
    frames: None, or host integers, one per utterance in [1, T]: utterance b is its first frames[b] frames (nothing
    later is read); z, zn are 0 from frame frames[b] on, Rss, Rnn and W from block ceil(frames[b] / block) on."""
    Rss, Rnn = ops.scm_recursive(Y, mask, Z, lambda_cor, block, power, R0, n_fft, frames=frames)
    W, _ = ops.mwf_solve(Rss, Rnn, mu, filter_type, rank)
    W = _live_blocks(W, frames, Y.shape[3], block)
    z, zn = ops.filter_sum_blocks(W, Y, Z, block, lag, True, ref, n_fft, frames=frames)
    return {"z": z, "zn": zn, "W": W, "Rss": Rss, "Rnn": Rnn}


def _online_mwf_split(Y, Xs, Xn, Z, Zs, Zn, mask, lambda_cor, block, lag, mu, filter_type, rank, ref, R0, n_fft,
                      frames):
    """online_mwf with the speech and noise statistics read from their own channel stacks: R_ss is the unweighted
    recursive scan of [Xs ; Zs], R_nn that of [Xn ; Zn], each seeded by its half of R0, and the filters apply to
    [Y ; Z].  With a mask, Xs and Xn are first scaled by mask and 1 - mask (the own channels of a step 2 whose other
    nodes contribute z_rs / z_rn, as in tango.tango_step2).  Returns dict(z, zn, W, Rss, Rnn) as online_mwf."""
    if mask is not None:
        Xs, Xn = ops.apply_mask(Xs, mask, False), ops.apply_mask(Xn, mask, True)
    r0s, r0n = (None, None) if R0 is None else ((R0[0], R0[0]), (R0[1], R0[1]))   # the second matrix is not used
    Rss, _ = ops.scm_recursive(Xs, None, Zs, lambda_cor, block, 2, r0s, n_fft, frames=frames)
    Rnn, _ = ops.scm_recursive(Xn, None, Zn, lambda_cor, block, 2, r0n, n_fft, frames=frames)
    W, _ = ops.mwf_solve(Rss, Rnn, mu, filter_type, rank)
    W = _live_blocks(W, frames, Y.shape[3], block)
    z, zn = ops.filter_sum_blocks(W, Y, Z, block, lag, True, ref, n_fft, frames=frames)
    return {"z": z, "zn": zn, "W": W, "Rss": Rss, "Rnn": Rnn}


def _uneven_batch(y, lens, n_fft):
    """The spectra of an uneven batch (stft_lengths: 0 past each utterance's frames), its per-utterance frame counts
    and the clip that sets a mask to 0 past them (a selection: a NaN there stays out of the statistics)."""
    Y = ops.stft_lengths(y, lens, n_fft)
    return Y, ops.n_frames(lens, n_fft), _frame_clip(lens, Y.shape[3], n_fft, Y.device)


def _clean_spectra(s, n, lens, n_fft):
    """S, N [B, K, C, T, F] of the clean components, one transform each as tango_batched takes them (the STFT pairs
    signals 2p, 2p + 1 of one call, so the grouping decides the bits)."""
    if lens is None:
        return ops.stft(s, n_fft), ops.stft(n, n_fft)
    return ops.stft_lengths(s, lens, n_fft), ops.stft_lengths(n, lens, n_fft)


def _filtered_pair(W, S, N, Zs, Zn, block, lag, ref, n_fft, frames):
    """The block filters W applied to the clean components: W^H [S ; Zs] and W^H [N ; Zn] [B, K, T, F], channel ref
    passed through before the first filter, as filter_sum_blocks does for the mixture."""
    return (ops.filter_sum_blocks(W, S, Zs, block, lag, True, ref, n_fft, frames=frames)[0],
            ops.filter_sum_blocks(W, N, Zn, block, lag, True, ref, n_fft, frames=frames)[0])


def online_tango(y, masks=None, lambda_cor=0.95, block=8, lag=1, mu=1.0, rank=1, ref_mic=0, n_fft=512, R0=None,
                 lengths=None, *, s=None, n=None, vads=("irm1", "irm1"), mask_for_z="local", filter_type="gevd",
                 diagnostics=True):
    """Two-step recursive Tango on time signals y [B, K, C, L]: local recursive MWF -> exchange of the compressed
    signals z -> recursive MWF on [own mics ; z of the other nodes] (the channel order of concatenate_signals,
    tango.py:142-155).  masks = (mask_z, mask_w) [B, K, T, F] frame-major (mask_w None: mask_z; or a callable
    mask_w(Y, z_y, zn) -> [B, K, T, F] called after step 1); R0 = optional initial (R_ss, R_nn) of the local step
    [B, K, F, C, C] (the second step of a multi-node array starts from zeros).  Returns yf, z_y, zn [B, K, T, F] and
    the per-block filters W1, W2.

    s, n: the clean components [B, K, C, L] float32 of y (the module docstring states what they add).  masks=None
    builds the masks of vads from them, mask_for_z selects the exchange mode, filter_type / mu / rank reach both
    solves, and with diagnostics the output also holds z_s, z_n, sf, nf; with masks=None, masks_z and mask_w as well.
    The argument errors of tango_batched are raised before any device work.  Without s, n and with the default
    options the call is the bare deployment step.

    lengths: None, or one length in samples per utterance, n_fft / 2 < lengths[b] <= L (as tango_batched takes
    them).  Utterance b is then y[b, ..., :lengths[b]] with T_b = 1 + lengths[b] // hop frames (s, n likewise): its
    outputs are those of the utterance run alone on frames t < T_b and 0 from T_b on, its W1, W2 those of the lone
    run on blocks j < ceil(T_b / block) and 0 after; masks past T_b are ignored.  Bit-identical to the lone run when
    K * C is even (the STFT transforms signals 2p, 2p + 1 together; DESIGN §5).  post.to_time(out, L,
    layout="TF", lengths=lengths) turns the outputs into signals per utterance."""
    _check_sources(masks, s, n, vads, mask_for_z)
    lens = _uneven_lengths(lengths, y.shape[0], y.shape[-1], n_fft)   # None: the uniform batch
    frames = clip = None
    if lens is None:
        Y = ops.stft(y, n_fft)
    else:
        Y, frames, clip = _uneven_batch(y, lens, n_fft)
    have_sn = s is not None and n is not None
    S = N = None
    if have_sn and (masks is None or diagnostics or "use_oracle_" in mask_for_z or mask_for_z == "compressed"):
        S, N = _clean_spectra(s, n, lens, n_fft)
    if masks is None:
        mask_z, mask_w = _clean_masks(S, N, s, vads, ref_mic, n_fft, lens)
    else:
        mask_z, mask_w = masks
        mask_w = mask_z if mask_w is None else mask_w
    if clip is not None:
        mz = clip(mask_z)
        mask_w = mz if mask_w is mask_z else (mask_w if callable(mask_w) else clip(mask_w))
        mask_z = mz
    K = Y.shape[1]
    opts = (lambda_cor, block, lag, mu, filter_type, rank, ref_mic)
    if "use_oracle_" in mask_for_z:
        s1 = _online_mwf_split(Y, S, N, None, None, None, None, *opts, R0, n_fft, frames)
    else:
        s1 = online_mwf(Y, mask_z, None, *opts, 2, R0, n_fft, frames)
    z_y = s1["z"]
    if callable(mask_w):
        mask_w = mask_w(Y, z_y, s1["zn"])
        if clip is not None:
            mask_w = clip(mask_w)
    z_s = z_n = None
    if have_sn and (diagnostics or mask_for_z in ("compressed", "use_oracle_zs")):
        z_s, z_n = _filtered_pair(s1["W"], S, N, None, None, block, lag, ref_mic, n_fft, frames)
    z_rs, z_rn = _z_for_stats(mask_for_z, vads, z_y, mask_w, z_s, z_n,
                              lambda: (_ref_plane(S, ref_mic), _ref_plane(N, ref_mic)), clip)
    # a single node has no other nodes: step 2 reads its own channels only and starts from R0 like step 1
    Z, R2 = (None, R0) if K == 1 else (z_y, None)
    if z_rs is None:
        s2 = online_mwf(Y, mask_w, Z, *opts, 2, R2, n_fft, frames)
    else:
        s2 = _online_mwf_split(Y, Y, Y, Z, *((None, None) if K == 1 else (z_rs, z_rn)), mask_w, *opts, R2, n_fft,
                               frames)
    out = {"yf": s2["z"], "z_y": z_y, "zn": s1["zn"], "W1": s1["W"], "W2": s2["W"]}
    if have_sn and diagnostics:
        out["sf"], out["nf"] = _filtered_pair(s2["W"], S, N, *((None, None) if K == 1 else (z_s, z_n)), block, lag,
                                              ref_mic, n_fft, frames)
        out["z_s"], out["z_n"] = z_s, z_n
    if masks is None:
        out["masks_z"], out["mask_w"] = mask_z, mask_w
    return out
