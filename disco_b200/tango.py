"""Two-step distributed MWF ("Tango") on the GPU, batched over utterances.

``tango_batched`` is the native entry point: device tensors in, device tensors out, every array
node of every utterance processed by the same handful of kernel launches.  ``offline_tango`` keeps
the reference signature (disco_theque/speech_enhancement/tango.py:252) on NumPy lists and is a thin
adapter over it.

Step 1 (reference tango.py:326-376), per group g = (utterance b, node k):
    Y, R_ss, R_nn = stft_scm(y, mask_z)      fused STFT + masked SCM         (kernel stft_scm)
    w             = mwf_solve(R_ss, R_nn)    rank-1 GEVD-MWF per bin          (kernel mwf_solve)
    z, zn         = filter_sum(w, Y)         z = w^H Y, zn = Y[ref] - z       (kernel filter_sum)
Exchange (reference tango.py:379-386): every node needs the z of all other nodes.  Inside one
GPU that is just the Z[b, :, :, :] tensor; when nodes are sharded over GPUs it is an all-gather
(disco_b200/dist.py).
Step 2 (reference tango.py:411-450), per group: the D = C + K - 1 channels [Y_k ; z_{j != k}] are
never concatenated in memory -- the kernels index Y and Z directly:
    R_ss, R_nn = masked_scm(Y, Z, mask_w);  w = mwf_solve(...);  yf = filter_sum(w, Y, Z)
"""
import numpy as np
import torch

from . import ops

OUTPUT_NAMES = ("yf", "sf", "nf", "z_y", "z_s", "z_n", "zn", "masks_z", "mask_w")


def _ref_plane(X, ref):
    """X [B, K, C, T, F] -> contiguous [B, K, T, F] plane of channel `ref`."""
    return X[:, :, ref].contiguous()


def _bcast_mask(X, m, one_minus):
    """m (or 1 - m) [B, K, T, F] applied to every channel of X [B, K, C, T, F] (one launch)."""
    return ops.apply_mask(X, m, one_minus)


def _ivad_mask(s_ref, n_fft, lengths=None):
    """'ivad' masks (tango.py:216-221): the per-sample energy VAD of the clean reference channel,
    taken every hop and spread over all bins.  s_ref [B, K, L] -> [B, K, T, F] float32 (0/1); all (b, k) at once.
    lengths [B] (host, or None): utterance b is its first lengths[b] samples, so its VAD (quantile and framing) is
    taken over those alone, once per distinct length, and its frames from 1 + lengths[b] // hop on are 0."""
    from .compat.sigproc_utils import vad_oracle_rows_device
    B, K, L = s_ref.shape
    hop, F, T = n_fft // 2, n_fft // 2 + 1, ops.n_frames(L, n_fft)
    out = torch.zeros((B, K, T, F), dtype=torch.float32, device=s_ref.device)
    if lengths is None:
        vad = vad_oracle_rows_device(s_ref.reshape(B * K, L), win_len=n_fft, win_hop=hop)[:, ::hop]  # [B*K, <= T]
        out[:, :, :vad.shape[1], :] = vad.to(torch.float32).view(B, K, -1, 1)
        return out
    for Lb in sorted({int(v) for v in lengths}):
        idx = torch.from_numpy(np.flatnonzero(np.asarray(lengths) == Lb)).to(s_ref.device)
        rows = s_ref.index_select(0, idx)[..., :Lb]
        vad = vad_oracle_rows_device(rows.reshape(-1, Lb), win_len=n_fft, win_hop=hop)[:, ::hop]
        out[idx, :, :vad.shape[1], :] = vad.to(torch.float32).view(len(idx), K, -1, 1)
    return out


def _uneven_lengths(lengths, B, L, n_fft):
    """Host int32 [B] lengths of a batch whose utterances do not all have L samples; None for lengths=None or all L
    (the uniform batch)."""
    if lengths is None:
        return None
    host = ops.signal_lengths(lengths, (B,), L, lo=n_fft // 2)
    return None if bool((host == L).all()) else host


def _frame_clip(lengths, T, n_fft, device):
    """m -> m with every frame t >= 1 + lengths[b] // hop of utterance b set to 0, for [B, K, T, F] masks (a selection,
    so that a 0/0 = NaN of an oracle mask on the zero frames past the end is replaced, not multiplied)."""
    Tb = torch.from_numpy(1 + np.asarray(lengths, dtype=np.int64) // (n_fft // 2)).to(device)
    past = (torch.arange(T, device=device)[None, :] >= Tb[:, None]).view(-1, 1, T, 1)
    return lambda m: m.masked_fill(past, 0.0)


# network masks see windows of 21 frames, hop 1, and predict the middle one (reference tango.py:34-35, 340)
_DNN_WINDOW = dict(win_len=21, win_hop=1, frame_to_pred="mid")


def _mask_kind(vad):
    """'oracle' ('irmX' / 'ibmX' / 'iamX'), 'ivad' or 'dnn' ('crnn' / 'rnn'), as get_mask tells them apart
    (tango.py:189-223)."""
    if isinstance(vad, str) and len(vad) == 4 and vad[:3] in ("irm", "ibm", "iam") and vad[3].isdigit():
        return "oracle"
    if vad in ("ivad", "crnn", "rnn"):
        return "ivad" if vad == "ivad" else "dnn"
    raise ValueError("Unknown value for `mask_type`")                  # tango.py:223


def _z_for_mask(k, K, z_sigs):
    """The compressed signals that feed node k's step-2 mask estimator, in the order of get_z_for_mask
    (tango.py:158-186): (signal, node) pairs, signal 0 = z_y and 1 = zn.  'zs_hat' / 'zn_hat' take that signal of
    every other node; any other z_sigs takes z_y, zn of every other node in turn."""
    others = [j for j in range(K) if j != k]
    if z_sigs in ("zs_hat", "zn_hat"):
        return [(int(z_sigs == "zn_hat"), j) for j in others]
    return [(t, j) for j in others for t in (0, 1)]


def _dnn_masks(mod, Y0, z=None, nodes=None, z_sigs="zs_hat"):
    """Masks `mod` predicts on the device (tango.py:209-215) from Y0 [B, n, T, F], the mixture spectrum of the
    microphone each estimator listens to, for the nodes `nodes` of the array (default 0 .. n-1).  With
    z = (z_y, zn) [B, K, T, F] the estimator of node k also hears _z_for_mask(k, K, z_sigs).  -> [B, n, T, F]."""
    from . import dnn_mask
    B, n, T, F = Y0.shape
    nodes = range(n) if nodes is None else nodes
    ft = lambda a: a.transpose(-1, -2)                                  # frame-major [T, F] -> (F, T) view
    out = []
    for b in range(B):
        for i, k in enumerate(nodes):
            zl = None if z is None else [ft(z[t][b, j]) for t, j in _z_for_mask(k, z[0].shape[1], z_sigs)]
            out.append(dnn_mask.estimate_mask(mod, ft(Y0[b, i]), zl, device=Y0.device, **_DNN_WINDOW))
    return torch.stack(out).view(B, n, T, F)


def _step1_mask(vad, mods, ref_spectra, s_ref, y_ref, n_fft, lengths=None):
    """Step-1 mask [B, K, T, F] of the reference microphone (tango.py:338-342): an oracle type of its clean
    spectra ref_spectra() -> (S_ref, N_ref), 'ivad' of its clean signal s_ref [B, K, L], or mods[0] on its mixture
    spectrum y_ref() [B, K, T, F].  The spectra are callables so that each caller keeps its own STFT grouping
    (the two-for-one FFT makes a channel's bits depend on its partner signal) and computes only what `vad` needs.
    lengths: per-utterance lengths of an uneven batch (for 'ivad'), or None."""
    kind = _mask_kind(vad)
    if kind == "ivad":                                                  # tango.py:216-221
        return _ivad_mask(s_ref, n_fft, lengths)
    if kind == "dnn":
        return _dnn_masks(mods[0], y_ref())
    return ops.tf_mask(*ref_spectra(), vad)


def _step2_mask(vads, mods, mask_z, ch0_spectra, s0, n_fft, Y0=None, z=None, nodes=None, z_sigs="zs_hat",
                ref_mic=0, lengths=None):
    """Step-2 mask [B, n, T, F] (tango.py:387-394).  mask_z itself for the step-1 oracle kind on the same
    microphone, or for a network step without a model of its own (mods[1] None, tango.py:388-389); otherwise an
    oracle type or 'ivad' of microphone 0 (ch0_spectra, s0 as in _step1_mask) or mods[1] on Y0 [B, n, T, F]
    (microphone 0 of the nodes `nodes`) and the compressed signals z = (z_y, zn) chosen by z_sigs."""
    if _mask_kind(vads[1]) == "dnn":
        return mask_z if mods[1] is None else _dnn_masks(mods[1], Y0, z, nodes, z_sigs)
    if vads[1] == vads[0] and ref_mic == 0:
        return mask_z
    return _step1_mask(vads[1], None, ch0_spectra, s0, None, n_fft, lengths)


def _check_sources(masks, s, n, vads, mask_for_z):
    """The argument errors of an entry point that takes masks or the clean components s, n (tango_batched,
    online.online_tango), raised before any device work."""
    if mask_for_z is None:
        raise TypeError("argument of type 'NoneType' is not iterable")   # reference tango.py:343
    if masks is None and (s is None or n is None):
        raise ValueError("either masks or the clean components (s, n) are required")
    if (s is None or n is None) and mask_for_z in ("compressed", "use_oracle_refs", "use_oracle_zs"):
        raise ValueError("mask_for_z=%r needs the clean components s and n" % mask_for_z)
    if masks is None and "dnn" in [_mask_kind(v) for v in vads]:
        raise ValueError("network masks ('crnn' / 'rnn') come in through masks=")
    if mask_for_z == "use_oracle_sigs":
        raise NotImplementedError(_ORACLE_SIGS)


def _clean_masks(S, N, s, vads, ref_mic, n_fft, lengths=None):
    """(mask_z, mask_w) [B, K, T, F] of the clean components: vads[0] of microphone ref_mic and vads[1] of microphone 0
    (mask_z itself where they coincide) from their spectra S, N [B, K, C, T, F] or, for 'ivad', the signal s."""
    spectra = lambda ch: (_ref_plane(S, ch), _ref_plane(N, ch))
    mask_z = _step1_mask(vads[0], None, lambda: spectra(ref_mic), s[:, :, ref_mic], None, n_fft, lengths)
    return mask_z, _step2_mask(vads, None, mask_z, lambda: spectra(0), s[:, :, 0], n_fft, ref_mic=ref_mic,
                               lengths=lengths)


_ORACLE_SIGS = "'use_oracle_sigs' is ill-formed in the reference (tango.py:423-427 indexes per-channel arrays by node)"


def _z_for_stats(mask_for_z, vads, Z, mask_w, Zs, Zn, oracle_refs, clip=None):
    """What the other nodes contribute to the step-2 speech / noise statistics (tango.py:396-429): (z_rs, z_rn)
    [B, K, T, F] from the compressed signals Z, the step-2 masks mask_w, the filtered clean components Zs, Zn and
    oracle_refs() -> clean spectra of the reference microphones; (None, None) for 'local', where z is masked by
    the step-2 mask of the node being filtered.  clip: zeroes the frames past each utterance's end of a mask
    (uneven batches), or None."""
    if mask_for_z == "local":
        return None, None
    if mask_for_z == "distant":
        return ops.apply_mask(Z, mask_w, False), ops.apply_mask(Z, mask_w, True)
    if mask_for_z == "compressed":
        mc = ops.tf_mask(Zs, Zn, vads[0])
        if clip is not None:
            mc = clip(mc)
        return ops.apply_mask(Z, mc, False), ops.apply_mask(Z, mc, True)
    if mask_for_z == "use_oracle_refs":
        return oracle_refs()
    if mask_for_z == "use_oracle_zs":
        return Zs, Zn
    if mask_for_z == "use_oracle_sigs":
        raise NotImplementedError(_ORACLE_SIGS)
    return Z, Z              # 'previous' and any other string: unmasked z in both statistics (tango.py:428-429)


def _reference_lists(res, names, vads, masks=None):
    """res[name] [K, ...] NumPy arrays -> the reference's lists of K arrays, one per name.  Like the reference,
    oracle 'ibmX' masks are bool and 'ivad' masks float64; externally supplied masks stay float32."""
    out = []
    for nm in names:
        arr = res[nm]
        vad = {"masks_z": vads[0], "mask_w": vads[1]}.get(nm) if masks is None else None
        if vad is not None and "ibm" in vad:
            arr = arr.astype(bool)
        elif vad == "ivad":
            arr = arr.astype(np.float64)
        out.append([arr[k] for k in range(len(arr))])
    return tuple(out)


def tango_step1(y, mask_z, n_fft=512, mu=1.0, filter_type="gevd", rank=1, ref_mic=0, oracle_sn=None,
                apply_filter=True, lengths=None):
    """y [B, K, C, L] float32, mask_z [B, K, T, F] float32 (frame-major).
    Returns dict: Y [B,K,C,T,F], z_y, zn [B,K,T,F], W1 [B,K,F,C], R_ss, R_nn.
    oracle_sn = (S, N) spectra replaces the masked estimates in the SCMs ('use_oracle_*', tango.py:343-345).
    apply_filter=False leaves z_y / zn to a fused later pass (single-node arrays).
    lengths [B] (host ints, or None): utterances of their own lengths; Y is then stft_lengths' (zero past each
    utterance's frames) and the matrices are the sums over its frames divided by T = 1 + L // hop, not by its own
    frame count (a common scale of R_ss and R_nn, which the filters do not depend on)."""
    B, K, C, L = y.shape
    T, F = ops.n_frames(L, n_fft), n_fft // 2 + 1
    fused = oracle_sn is None and lengths is None and ops.stft_scm_supported(n_fft, C, 1)
    if fused and C <= 4:
        # fused STFT + SCM; the solve reads the per-segment partial sums directly (no finalize launch)
        Y, ws = ops.stft_scm(y.view(B * K, C, L), mask_z.view(B * K, T, F), n_fft, keep_partials=True)
        Y = Y.view(B, K, C, T, F)
        W1, _ = ops.mwf_solve_workspace(ws, B * K, C, L, n_fft, mu, filter_type, rank)
        W1 = W1.view(B, K, F, C)
        z_y = zn = None
        if apply_filter:
            z_y, zn = ops.filter_sum(W1, Y, None, conj=True, ref=ref_mic, n_fft=n_fft)
        return {"Y": Y, "z_y": z_y, "zn": zn, "W1": W1, "R_ss": None, "R_nn": None}
    elif fused:
        # 5..8 microphones: same single pass, matrices materialised for the cooperative solver
        Y, Rss, Rnn = ops.stft_scm(y.view(B * K, C, L), mask_z.view(B * K, T, F), n_fft)
        Y, Rss, Rnn = Y.view(B, K, C, T, F), Rss.view(B, K, F, C, C), Rnn.view(B, K, F, C, C)
    else:
        Y = ops.stft(y, n_fft) if lengths is None else ops.stft_lengths(y, lengths, n_fft)
        if oracle_sn is None:
            Rss, Rnn = ops.masked_scm(Y, mask_z, None, n_fft)
        else:
            Rss, _ = ops.masked_scm(oracle_sn[0], None, None, n_fft)
            Rnn, _ = ops.masked_scm(oracle_sn[1], None, None, n_fft)
    W1, _ = ops.mwf_solve(Rss, Rnn, mu, filter_type, rank)
    z_y = zn = None
    if apply_filter:
        z_y, zn = ops.filter_sum(W1, Y, None, conj=True, ref=ref_mic, n_fft=n_fft)
    return {"Y": Y, "z_y": z_y, "zn": zn, "W1": W1, "R_ss": Rss, "R_nn": Rnn}


def tango_step2(Y, Z, mask_w, n_fft=512, mu=1.0, filter_type="gevd", rank=1, out_layout="TF", node_sel=None,
                z_rs=None, z_rn=None, z_layout="BK"):
    """Y [B, Ksel, C, T, F], Z [B, K, T, F] (all nodes' compressed signals), mask_w [B, Ksel, T, F].
    mask_for_z='local' when z_rs / z_rn are None; otherwise they are the [B, K, T, F] signals the
    other nodes contribute to the speech / noise statistics (own channels are still masked by mask_w).
    z_layout='KB': Z (and z_rs / z_rn) are node-major [K, B, T, F], as an all-gather over node-owning ranks
    delivers them (disco_b200/dist.py).
    Returns yf [B, Ksel, ...], W2 [B, Ksel, F, D]."""
    if z_rs is None:
        Rss, Rnn = ops.masked_scm(Y, mask_w, Z, n_fft, node_sel=node_sel, z_layout=z_layout)
    else:
        Rss, _ = ops.masked_scm(_bcast_mask(Y, mask_w, False), None, z_rs, n_fft, node_sel=node_sel, z_layout=z_layout)
        Rnn, _ = ops.masked_scm(_bcast_mask(Y, mask_w, True), None, z_rn, n_fft, node_sel=node_sel, z_layout=z_layout)
    W2, _ = ops.mwf_solve(Rss, Rnn, mu, filter_type, rank)
    yf = ops.filter_sum(W2, Y, Z, conj=True, n_fft=n_fft, out_layout=out_layout, node_sel=node_sel, z_layout=z_layout)
    return yf, W2


def tango_batched(y, s=None, n=None, masks=None, vads=("irm1", "irm1"), mask_for_z="local", n_fft=512,
                  mu=1.0, filter_type="gevd", rank=1, ref_mic=0, out_layout="FT", diagnostics=True, lengths=None):
    """Batched two-step Tango.

    y [B, K, C, L] float32 CUDA tensor (K nodes of C microphones).  Masks come either from the
    oracle (s, n given: 'irmX' / 'ibmX' / 'iamX' of the reference channel, tango.py:338-342,
    391-394) or from ``masks=(mask_z, mask_w)`` -- [B, K, T, F] float32 device tensors in
    frame-major layout, e.g. straight out of a mask-estimation DNN (``mask_w=None`` reuses
    mask_z, tango.py:388-389).
    Returns a dict with the reference's outputs (tango.py:457) as [B, K, F, T] (out_layout='FT') or
    [B, K, T, F] ('TF') tensors: yf, z_y, zn, masks_z, mask_w and, with s/n and diagnostics, sf, nf,
    z_s, z_n.

    lengths: one length per utterance ([B] integers, n_fft/2 < lengths[b] <= L), or None.  Utterance b is then its
    first lengths[b] samples (y, s, n zero after them) and has T_b = 1 + lengths[b] // hop frames: its outputs are
    those of the utterance alone, trimmed, to rounding, and every output (masks included) is exactly 0 from frame
    T_b on.  Such a batch runs the routes that store the spectra (the fused STFT+SCM kernels assume one length);
    lengths=None or all lengths equal to L is the uniform batch, computed exactly as without the argument.
    """
    _check_sources(masks, s, n, vads, mask_for_z)
    B, K, C, L = y.shape
    T, F = ops.n_frames(L, n_fft), n_fft // 2 + 1
    lens = _uneven_lengths(lengths, B, L, n_fft)
    stft = (lambda a: ops.stft(a, n_fft)) if lens is None else (lambda a: ops.stft_lengths(a, lens, n_fft))
    clip = None if lens is None else _frame_clip(lens, T, n_fft, y.device)
    oracle = masks is None
    have_sn = s is not None and n is not None
    S = N = None
    if have_sn and (oracle or diagnostics or "use_oracle_" in mask_for_z or mask_for_z == "compressed"):
        S, N = stft(s), stft(n)
    # ---- masks
    if oracle:
        mask_z, mask_w = _clean_masks(S, N, s, vads, ref_mic, n_fft, lens)
    else:
        mask_z, mask_w = masks
        if mask_w is None:
            mask_w = mask_z
    if clip is not None:
        # past an utterance's end its spectra are 0 and an oracle mask 0/0: every mask is 0 there
        mz = clip(mask_z)
        mask_w = mz if mask_w is mask_z else (mask_w if callable(mask_w) else clip(mask_w))
        mask_z = mz
    # mask_w may be a callable (Y, z_y, zn) -> [B, K, T, F]: a step-2 mask estimator that looks at the
    # compressed signals of the other nodes (tango.py:387-394)
    mask_w_fn = mask_w if callable(mask_w) else None
    # ---- step 1
    osn = (S, N) if "use_oracle_" in mask_for_z else None
    # single-node arrays with both masks known: the step-2 statistics are taken over the same Y as the step-1
    # statistics (tango.py:431-440 with K = 1), so ONE pass accumulates both and ONE pass applies both filters
    single = (K == 1 and mask_for_z == "local" and mask_w_fn is None and osn is None)
    same_mask = single and mask_w is mask_z
    fuse_dual = single and not same_mask and lens is None and ops.stft_scm_supported(n_fft, C, 2)
    # otherwise for single-node arrays: the step-1 filter-and-sum and the step-2 SCM share one pass over Y
    fuse_mid = (single and not same_mask and not fuse_dual and C <= 8)
    # multi-node arrays: z of every node + the step-2 SCMs of every node in one pass over Y
    fuse_multi = (K > 1 and mask_for_z == "local" and mask_w_fn is None and osn is None
                  and ops.tango_mid_supported(C, K))
    final_layout = False          # z_y / zn / yf already in `out_layout`
    R2 = W2 = yf = None
    if fuse_dual:
        # Y is never stored: the filter pass transforms y again, which moves half the bytes of reading Y back
        x = y.view(B * K, C, L)
        _, ws = ops.stft_scm2(x, mask_z.view(B * K, T, F), mask_w.view(B * K, T, F), n_fft, want_Y=False)
        W12, _ = ops.mwf_solve_workspace2(ws, B * K, C, L, n_fft, mu, filter_type, rank)
        W1, W2 = W12[0].view(B, K, F, C), W12[1].view(B, K, F, C)
        z_y, zn, yf = ops.stft_filter_dual(x, W12[0], W12[1], ref=ref_mic, n_fft=n_fft, out_layout=out_layout)
        shape = (B, K) + tuple(z_y.shape[1:])
        z_y, zn, yf = z_y.view(shape), zn.view(shape), yf.view(shape)
        final_layout = True
    else:
        st1 = tango_step1(y, mask_z, n_fft, mu, filter_type, rank, ref_mic, oracle_sn=osn,
                          apply_filter=not (fuse_mid or fuse_multi), lengths=lens)
        Y, z_y, zn, W1 = st1["Y"], st1["z_y"], st1["zn"], st1["W1"]
        if mask_w_fn is not None:
            mask_w = mask_w_fn(Y, z_y, zn)
            if clip is not None:
                mask_w = clip(mask_w)
        if same_mask:
            # K = 1 and mask_w is mask_z (tango.py:388-389): the step-2 statistics ARE the step-1 statistics,
            # so w_glo = w_loc and yf = z
            W2 = W1
        elif fuse_mid:
            z_y, zn, Rss2, Rnn2 = ops.filter_sum_scm(W1, Y, mask_w, ref=ref_mic, n_fft=n_fft)
            R2 = (Rss2, Rnn2)
        elif fuse_multi:
            z_y, zn, Rss2, Rnn2 = ops.tango_mid(W1, Y, mask_w, ref=ref_mic, n_fft=n_fft)
            R2 = (Rss2, Rnn2)
    z_s = z_n = None
    if have_sn and (diagnostics or mask_for_z in ("compressed", "use_oracle_zs")):
        z_s = ops.filter_sum(W1, S, None, conj=True, n_fft=n_fft)
        z_n = ops.filter_sum(W1, N, None, conj=True, n_fft=n_fft)
    z_rs, z_rn = _z_for_stats(mask_for_z, vads, z_y, mask_w, z_s, z_n,
                              lambda: (_ref_plane(S, ref_mic), _ref_plane(N, ref_mic)), clip)
    # ---- step 2
    ft = ops._layout(out_layout) == ops.FT
    conv = ops.transpose_last2 if ft else (lambda a: a)
    if yf is not None:
        pass                                                  # fuse_dual: already filtered
    elif same_mask:
        yf = conv(z_y) if ft else z_y.clone()
    elif R2 is not None:
        W2, _ = ops.mwf_solve(R2[0], R2[1], mu, filter_type, rank)
        yf = ops.filter_sum(W2, Y, z_y if K > 1 else None, conj=True, n_fft=n_fft, out_layout=out_layout)
    else:
        yf, W2 = tango_step2(Y, z_y, mask_w, n_fft, mu, filter_type, rank, out_layout, z_rs=z_rs, z_rn=z_rn)
    out = {"yf": yf}
    if have_sn and diagnostics:
        out["sf"] = ops.filter_sum(W2, S, z_s, conj=True, n_fft=n_fft, out_layout=out_layout)
        out["nf"] = ops.filter_sum(W2, N, z_n, conj=True, n_fft=n_fft, out_layout=out_layout)
    out["z_y"], out["zn"] = (z_y, zn) if final_layout else (conv(z_y), conv(zn))
    if z_s is not None and diagnostics:
        out["z_s"], out["z_n"] = conv(z_s), conv(z_n)
    out["masks_z"] = conv(mask_z)
    out["mask_w"] = out["masks_z"] if mask_w is mask_z else conv(mask_w)
    return out


# ------------------------------------------------------------------------------------------------
# Reference-signature adapter (NumPy lists in / NumPy lists out)
# ------------------------------------------------------------------------------------------------
def _to_dev(sig_lists, nodes, device):
    arr = np.stack([np.stack([np.asarray(ch, dtype=np.float32) for ch in sig_lists[k]]) for k in nodes])
    return torch.from_numpy(arr).to(device)[None]          # [1, len(nodes), C, L]


def _to_mask(mlist, nodes, device):
    """(F, T) masks of the nodes `nodes` -> [1, len(nodes), T, F] float32 on the device."""
    arr = np.stack([np.asarray(mlist[k], dtype=np.float32) for k in nodes])[None]   # [1, n, F, T]
    return ops.transpose_last2(torch.from_numpy(np.ascontiguousarray(arr)).to(device))


def offline_tango(y, s, n, vads="irm1", mods=None, mask_for_z="local", z_sigs="zs_hat", *,
                  n_fft=512, mu=1, filter_type="gevd", rank=1, masks=None, device="cuda"):
    """Drop-in for disco_theque.speech_enhancement.tango.offline_tango (tango.py:252-457).

    y, s, n: [node][channel] 1-D float32 signals (ragged channel counts allowed).  Returns the
    reference's 9 lists (length K) of (F, T) arrays: yf, sf, nf, z_y, z_s, z_n, zn (complex64),
    masks_z, mask_w (float32; bool for 'ibmX' and float64 for 'ivad' like the reference).
    Keyword-only extensions: n_fft, mu, filter_type, rank (module constants / literals in the
    reference) and masks=(mask_z[K], mask_w[K]) of (F, T) arrays for externally estimated masks.
    DNN mask types ('crnn') run ``mods`` on the device through disco_b200.dnn_mask.
    """
    if mask_for_z is None:
        raise TypeError("argument of type 'NoneType' is not iterable")   # reference tango.py:343
    if isinstance(vads, str):
        vads = [vads, vads]                                   # get_z_signals.py:279 passes one string
    dev = torch.device(device)
    if len({len(chans) for chans in y}) != 1:
        res = _offline_tango_ragged(y, s, n, vads, mods, mask_for_z, z_sigs, masks, n_fft, mu, filter_type, rank, dev)
        return _reference_lists(res, OUTPUT_NAMES, vads, masks)
    nodes = list(range(len(y)))
    yd, sd, nd = _to_dev(y, nodes, dev), _to_dev(s, nodes, dev), _to_dev(n, nodes, dev)
    mk = None
    if masks is not None:
        mk = (_to_mask(masks[0], nodes, dev), _to_mask(masks[1], nodes, dev))
    elif "dnn" in [_mask_kind(v) for v in vads]:
        # an oracle mask next to a network one is taken from an STFT of microphone 0 alone
        mic0 = lambda: (ops.stft(sd[:, :, 0].contiguous(), n_fft), ops.stft(nd[:, :, 0].contiguous(), n_fft))
        mask_z = _step1_mask(vads[0], mods, mic0, sd[:, :, 0], lambda: ops.stft(yd[:, :, 0].contiguous(), n_fft),
                             n_fft)
        # the step-2 estimator hears the other nodes' compressed signals: tango_batched calls it after step 1
        mk = (mask_z, lambda Y, z_y, zn: _step2_mask(vads, mods, mask_z, mic0, sd[:, :, 0], n_fft, Y[:, :, 0],
                                                     (z_y, zn), z_sigs=z_sigs))
    res = tango_batched(yd, sd, nd, masks=mk, vads=vads, mask_for_z=mask_for_z, n_fft=n_fft, mu=mu,
                        filter_type=filter_type, rank=rank, out_layout="FT")
    return _reference_lists({k: v[0].cpu().numpy() for k, v in res.items()}, OUTPUT_NAMES, vads, masks)


def _offline_tango_ragged(y, s, n, vads, mods, mask_for_z, z_sigs, masks, n_fft, mu, filter_type, rank, dev):
    """Nodes with different microphone counts (reference tango.py:259-260, 284): step 1 and step 2 run
    once per channel count on the nodes that have it; Z (and the signals the other nodes contribute to the
    step-2 statistics under every `mask_for_z` mode, tango.py:396-429) always hold all K nodes.  The mask
    estimators only see microphone 0 and the compressed signals, so they do not care about the channel counts.
    Returns the outputs as [K, F, T] NumPy arrays."""
    K = len(y)
    T, F = ops.n_frames(len(y[0][0]), n_fft), n_fft // 2 + 1
    groups = {}
    for k in range(K):
        groups.setdefault(len(y[k]), []).append(k)
    # all K nodes: Z = z_y, ZN = zn, Zs / Zn = z_s / z_n, Sref / Nref = clean spectra of microphone 0
    Z, ZN, Zs, Zn, Sref, Nref = (torch.empty((1, K, T, F), dtype=torch.complex64, device=dev) for _ in range(6))
    MZ = torch.empty((1, K, T, F), dtype=torch.float32, device=dev)
    MW = torch.empty_like(MZ)
    use_osn = "use_oracle_" in mask_for_z
    keep = []
    # ---- step 1 per channel count
    for C, nodes in sorted(groups.items()):
        yd, sd, nd = _to_dev(y, nodes, dev), _to_dev(s, nodes, dev), _to_dev(n, nodes, dev)
        S, N = ops.stft(sd, n_fft), ops.stft(nd, n_fft)
        idx = torch.tensor(nodes, device=dev)
        Sref[0, idx], Nref[0, idx] = S[0, :, 0], N[0, :, 0]
        if masks is not None:
            mz = _to_mask(masks[0], nodes, dev)
        else:
            mz = _step1_mask(vads[0], mods, lambda: (_ref_plane(S, 0), _ref_plane(N, 0)), sd[:, :, 0],
                             lambda: ops.stft(yd[:, :, 0].contiguous(), n_fft), n_fft)
        st1 = tango_step1(yd, mz, n_fft, mu, filter_type, rank, 0, oracle_sn=(S, N) if use_osn else None)
        zs = ops.filter_sum(st1["W1"], S, None, conj=True, n_fft=n_fft)
        zn = ops.filter_sum(st1["W1"], N, None, conj=True, n_fft=n_fft)
        Z[0, idx], Zs[0, idx], Zn[0, idx], ZN[0, idx] = st1["z_y"][0], zs[0], zn[0], st1["zn"][0]
        MZ[0, idx] = mz[0]
        keep.append((nodes, idx, st1["Y"], S, N, sd))
    # ---- step-2 masks, once every node's compressed signals exist
    for nodes, idx, Y, S, N, sd in keep:
        if masks is not None:
            MW[0, idx] = _to_mask(masks[1], nodes, dev)[0]
        else:
            MW[0, idx] = _step2_mask(vads, mods, MZ[:, idx], lambda: (_ref_plane(S, 0), _ref_plane(N, 0)),
                                     sd[:, :, 0], n_fft, Y[:, :, 0], (Z, ZN), nodes, z_sigs)[0]
    z_rs, z_rn = _z_for_stats(mask_for_z, vads, Z, MW, Zs, Zn, lambda: (Sref, Nref))
    # ---- step 2 per channel count
    res = {nm: np.empty((K, F, T), np.complex64) for nm in ("yf", "sf", "nf")}
    for nodes, idx, Y, S, N, sd in keep:
        yf, W2 = tango_step2(Y, Z, MW[:, idx].contiguous(), n_fft, mu, filter_type, rank, "FT", node_sel=nodes,
                             z_rs=z_rs, z_rn=z_rn)
        sf = ops.filter_sum(W2, S, Zs, conj=True, n_fft=n_fft, out_layout="FT", node_sel=nodes)
        nf = ops.filter_sum(W2, N, Zn, conj=True, n_fft=n_fft, out_layout="FT", node_sel=nodes)
        res["yf"][nodes], res["sf"][nodes], res["nf"][nodes] = yf[0].cpu().numpy(), sf[0].cpu().numpy(), \
            nf[0].cpu().numpy()
    tr = lambda a: ops.transpose_last2(a)[0].cpu().numpy()
    res.update(z_y=tr(Z), z_s=tr(Zs), z_n=tr(Zn), zn=tr(ZN), masks_z=tr(MZ), mask_w=tr(MW))
    return res
