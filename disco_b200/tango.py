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
_KNOWN_MASK_FOR_Z = ("local", "distant", "compressed", "use_oracle_refs", "use_oracle_zs", "previous")


def _is_oracle_type(t):
    return isinstance(t, str) and len(t) == 4 and t[:3] in ("irm", "ibm", "iam") and t[3].isdigit()


def _ref_plane(X, ref):
    """X [B, K, C, T, F] -> contiguous [B, K, T, F] plane of channel `ref`."""
    return X[:, :, ref].contiguous()


def _bcast_mask(X, m, one_minus):
    """m (or 1 - m) [B, K, T, F] applied to every channel of X [B, K, C, T, F] (one launch)."""
    return ops.apply_mask(X, m, one_minus)


def _ivad_mask(s_ref, n_fft):
    """'ivad' masks (tango.py:216-221): the per-sample energy VAD of the clean reference channel,
    taken every hop and spread over all bins.  s_ref [B, K, L] -> [B, K, T, F] float32 (0/1); all (b, k) at once."""
    from .compat.sigproc_utils import vad_oracle_rows_device
    B, K, L = s_ref.shape
    hop, F, T = n_fft // 2, n_fft // 2 + 1, ops.n_frames(L, n_fft)
    vad = vad_oracle_rows_device(s_ref.reshape(B * K, L), win_len=n_fft, win_hop=hop)[:, ::hop]      # [B*K, <= T]
    out = torch.zeros((B, K, T, F), dtype=torch.float32, device=s_ref.device)
    out[:, :, :vad.shape[1], :] = vad.to(torch.float32).view(B, K, -1, 1)
    return out


def tango_step1(y, mask_z, n_fft=512, mu=1.0, filter_type="gevd", rank=1, ref_mic=0, oracle_sn=None,
                apply_filter=True):
    """y [B, K, C, L] float32, mask_z [B, K, T, F] float32 (frame-major).
    Returns dict: Y [B,K,C,T,F], z_y, zn [B,K,T,F], W1 [B,K,F,C], R_ss, R_nn.
    oracle_sn = (S, N) spectra replaces the masked estimates in the SCMs ('use_oracle_*', tango.py:343-345).
    apply_filter=False leaves z_y / zn to a fused later pass (single-node arrays)."""
    B, K, C, L = y.shape
    T, F = ops.n_frames(L, n_fft), n_fft // 2 + 1
    fused = oracle_sn is None and ops.stft_scm_supported(n_fft, C, 1)
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
        Y = ops.stft(y, n_fft)
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
                  mu=1.0, filter_type="gevd", rank=1, ref_mic=0, out_layout="FT", diagnostics=True):
    """Batched two-step Tango.

    y [B, K, C, L] float32 CUDA tensor (K nodes of C microphones).  Masks come either from the
    oracle (s, n given: 'irmX' / 'ibmX' / 'iamX' of the reference channel, tango.py:338-342,
    391-394) or from ``masks=(mask_z, mask_w)`` -- [B, K, T, F] float32 device tensors in
    frame-major layout, e.g. straight out of a mask-estimation DNN (``mask_w=None`` reuses
    mask_z, tango.py:388-389).
    Returns a dict with the reference's outputs (tango.py:457) as [B, K, F, T] (out_layout='FT') or
    [B, K, T, F] ('TF') tensors: yf, z_y, zn, masks_z, mask_w and, with s/n and diagnostics, sf, nf,
    z_s, z_n.
    """
    if mask_for_z is None:
        raise TypeError("argument of type 'NoneType' is not iterable")   # reference tango.py:343
    B, K, C, L = y.shape
    oracle = masks is None
    if oracle and (s is None or n is None):
        raise ValueError("either masks or the clean components (s, n) are required")
    have_sn = s is not None and n is not None
    if not have_sn and mask_for_z in ("compressed", "use_oracle_refs", "use_oracle_zs"):
        raise ValueError("mask_for_z=%r needs the clean components s and n" % mask_for_z)
    S = N = None
    if have_sn and (oracle or diagnostics or "use_oracle_" in mask_for_z):
        S, N = ops.stft(s, n_fft), ops.stft(n, n_fft)
    # ---- masks
    if oracle:
        for v in vads:
            if not (_is_oracle_type(v) or v == "ivad"):
                raise ValueError("Unknown value for `mask_type`")      # tango.py:223

        def oracle_mask(kind, ch):
            if kind == "ivad":                                          # tango.py:216-221
                return _ivad_mask(s[:, :, ch], n_fft)
            return ops.tf_mask(_ref_plane(S, ch), _ref_plane(N, ch), kind)
        mask_z = oracle_mask(vads[0], ref_mic)
        if vads[1] == vads[0] and ref_mic == 0:
            mask_w = mask_z
        else:
            mask_w = oracle_mask(vads[1], 0)                            # channel 0, tango.py:391
    else:
        mask_z, mask_w = masks
        if mask_w is None:
            mask_w = mask_z
    # mask_w may be a callable (Y, z_y, zn) -> [B, K, T, F]: a step-2 mask estimator that looks at the
    # compressed signals of the other nodes (tango.py:387-394)
    mask_w_fn = mask_w if callable(mask_w) else None
    # ---- step 1
    osn = (S, N) if "use_oracle_" in mask_for_z else None
    T, F = ops.n_frames(L, n_fft), n_fft // 2 + 1
    # single-node arrays with both masks known: the step-2 statistics are taken over the same Y as the step-1
    # statistics (tango.py:431-440 with K = 1), so ONE pass accumulates both and ONE pass applies both filters
    single = (K == 1 and mask_for_z == "local" and mask_w_fn is None and osn is None)
    same_mask = single and mask_w is mask_z
    fuse_dual = single and not same_mask and ops.stft_scm_supported(n_fft, C, 2)
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
                          apply_filter=not (fuse_mid or fuse_multi))
        Y, z_y, zn, W1 = st1["Y"], st1["z_y"], st1["zn"], st1["W1"]
        if mask_w_fn is not None:
            mask_w = mask_w_fn(Y, z_y, zn)
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
    # ---- what the other nodes contribute to the step-2 statistics (tango.py:396-429)
    z_rs = z_rn = None
    if mask_for_z == "local":
        pass
    elif mask_for_z == "distant":
        z_rs, z_rn = ops.apply_mask(z_y, mask_w, False), ops.apply_mask(z_y, mask_w, True)
    elif mask_for_z == "compressed":
        mc = ops.tf_mask(z_s, z_n, vads[0])
        z_rs, z_rn = ops.apply_mask(z_y, mc, False), ops.apply_mask(z_y, mc, True)
    elif mask_for_z == "use_oracle_refs":
        z_rs, z_rn = _ref_plane(S, ref_mic), _ref_plane(N, ref_mic)
    elif mask_for_z == "use_oracle_zs":
        z_rs, z_rn = z_s, z_n
    elif mask_for_z == "use_oracle_sigs":
        raise NotImplementedError("'use_oracle_sigs' is ill-formed in the reference (tango.py:423-427 "
                                  "indexes per-channel arrays by node)")
    else:   # 'previous' and any other string: unmasked z in both statistics (tango.py:428-429)
        z_rs = z_rn = z_y
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


def offline_tango(y, s, n, vads="irm1", mods=None, mask_for_z="local", z_sigs="zs_hat", *,
                  n_fft=512, mu=1, filter_type="gevd", rank=1, masks=None, device="cuda"):
    """Drop-in for disco_theque.speech_enhancement.tango.offline_tango (tango.py:252-457).

    y, s, n: [node][channel] 1-D float32 signals (ragged channel counts allowed).  Returns the
    reference's 9 lists (length K) of (F, T) arrays: yf, sf, nf, z_y, z_s, z_n, zn (complex64),
    masks_z, mask_w (float32; bool for 'ibmX' like the reference).
    Keyword-only extensions: n_fft, mu, filter_type, rank (module constants / literals in the
    reference) and masks=(mask_z[K], mask_w[K]) of (F, T) arrays for externally estimated masks.
    DNN mask types ('crnn') run ``mods`` on the device through disco_b200.dnn_mask.
    """
    if mask_for_z is None:
        raise TypeError("argument of type 'NoneType' is not iterable")   # reference tango.py:343
    if isinstance(vads, str):
        vads = [vads, vads]                                   # get_z_signals.py:279 passes one string
    K = len(y)
    chans = [len(y[k]) for k in range(K)]
    L = len(y[0][0])
    T, F = ops.n_frames(L, n_fft), n_fft // 2 + 1
    uniform = len(set(chans)) == 1
    use_dnn = masks is None and any("rnn" in v for v in vads)
    if use_dnn and uniform:
        return _offline_tango_dnn(y, s, n, vads, mods, mask_for_z, z_sigs, n_fft, mu, filter_type, rank,
                                  torch.device(device))
    dev = torch.device(device)

    def to_mask(mlist, nodes):
        arr = np.stack([np.asarray(mlist[k], dtype=np.float32) for k in nodes])[None]   # [1, n, F, T]
        return ops.transpose_last2(torch.from_numpy(np.ascontiguousarray(arr)).to(dev))

    if uniform:
        nodes = list(range(K))
        mk = None if masks is None else (to_mask(masks[0], nodes), to_mask(masks[1], nodes))
        res = tango_batched(_to_dev(y, nodes, dev), _to_dev(s, nodes, dev), _to_dev(n, nodes, dev), masks=mk,
                            vads=vads, mask_for_z=mask_for_z, n_fft=n_fft, mu=mu, filter_type=filter_type,
                            rank=rank, out_layout="FT")
        res = {k: v[0].cpu().numpy() for k, v in res.items()}
    else:
        res = _offline_tango_ragged(y, s, n, vads, mask_for_z, n_fft, mu, filter_type, rank, masks, dev, to_mask,
                                    mods=mods, z_sigs=z_sigs)
    is_bool = [masks is None and "ibm" in v for v in vads]
    is_f64 = [masks is None and v == "ivad" for v in vads]       # the reference's VAD masks are float64
    out = []
    for nm in OUTPUT_NAMES:
        arr = res[nm]
        if nm == "masks_z" and is_bool[0] or nm == "mask_w" and is_bool[1]:
            arr = arr.astype(bool)
        if nm == "masks_z" and is_f64[0] or nm == "mask_w" and is_f64[1]:
            arr = arr.astype(np.float64)
        out.append([arr[k] for k in range(K)])
    return tuple(out)


def _offline_tango_dnn(y, s, n, vads, mods, mask_for_z, z_sigs, n_fft, mu, filter_type, rank, dev):
    """vads[i] == 'crnn' (or 'rnn'): masks predicted on the device by mods[i] (tango.py:209-215).
    Step 1 feeds |Y_ref| alone; step 2 feeds |Y_0| plus the compressed signals of the other nodes chosen by
    z_sigs (get_z_for_mask, tango.py:158-186); mods[1] is None with vads[1] == 'crnn' reuses the step-1 mask
    (tango.py:388-389).  Window length / predicted frame are the reference's constants (tango.py:34-35)."""
    from . import dnn_mask
    K = len(y)
    nodes = list(range(K))
    yd, sd, nd = _to_dev(y, nodes, dev), _to_dev(s, nodes, dev), _to_dev(n, nodes, dev)
    kw = dict(win_len=21, win_hop=1, frame_to_pred="mid", device=dev)
    spec_ft = lambda a: a.transpose(-1, -2)                         # frame-major [T, F] -> (F, T) view

    def oracle(kind, ch):
        S, N = ops.stft(sd[:, :, ch].contiguous(), n_fft), ops.stft(nd[:, :, ch].contiguous(), n_fft)
        return ops.tf_mask(S, N, kind)

    if "rnn" in vads[0]:
        Yref = ops.stft(yd[:, :, 0].contiguous(), n_fft)            # ref mic 0 (tango.py:338)
        mask_z = torch.stack([dnn_mask.estimate_mask(mods[0], spec_ft(Yref[0, k]), None, **kw) for k in nodes])[None]
    else:
        mask_z = oracle(vads[0], 0)

    def step2_mask(Y, z_y, zn):
        if "rnn" not in vads[1]:
            return oracle(vads[1], 0)
        if mods[1] is None:
            return mask_z
        out = []
        for k in nodes:
            others = [j for j in nodes if j != k]
            if z_sigs in ("zs_hat", "zn_hat"):
                zin = z_y if z_sigs == "zs_hat" else zn
                zl = [spec_ft(zin[0, j]) for j in others]
            else:                                                     # interleaved zs_j, zn_j of the other nodes
                zl = [spec_ft(t[0, j]) for j in others for t in (z_y, zn)]
            out.append(dnn_mask.estimate_mask(mods[1], spec_ft(Y[0, k, 0]), zl, **kw))
        return torch.stack(out)[None]

    res = tango_batched(yd, sd, nd, masks=(mask_z, step2_mask), vads=vads, mask_for_z=mask_for_z, n_fft=n_fft,
                        mu=mu, filter_type=filter_type, rank=rank, out_layout="FT")
    res = {k: v[0].cpu().numpy() for k, v in res.items()}
    return tuple([res[nm][k] for k in range(K)] for nm in OUTPUT_NAMES)


def _offline_tango_ragged(y, s, n, vads, mask_for_z, n_fft, mu, filter_type, rank, masks, dev, to_mask,
                          mods=None, z_sigs="zs_hat"):
    """Nodes with different microphone counts (reference tango.py:259-260, 284): step 1 and step 2 run
    once per channel count on the nodes that have it; Z (and the signals the other nodes contribute to the
    step-2 statistics under every `mask_for_z` mode, tango.py:396-429) always hold all K nodes.
    Masks: oracle types, externally supplied `masks`, or DNN masks (`mods`, tango.py:209-215) -- the estimators only
    see the reference microphone and the compressed signals, so they do not care about the channel counts."""
    if mask_for_z == "use_oracle_sigs":
        raise NotImplementedError("'use_oracle_sigs' is ill-formed in the reference (tango.py:423-427 "
                                  "indexes per-channel arrays by node)")
    K = len(y)
    L = len(y[0][0])
    T, F = ops.n_frames(L, n_fft), n_fft // 2 + 1
    dnn = masks is None and any("rnn" in v for v in vads)
    if dnn:
        from . import dnn_mask
        dkw = dict(win_len=21, win_hop=1, frame_to_pred="mid", device=dev)
    spec_ft = lambda a: a.transpose(-1, -2)
    groups = {}
    for k in range(K):
        groups.setdefault(len(y[k]), []).append(k)
    cplx = lambda: torch.empty((1, K, T, F), dtype=torch.complex64, device=dev)
    Z, Zs, Zn_, ZN, Sref, Nref, Yref = cplx(), cplx(), cplx(), cplx(), cplx(), cplx(), cplx()
    MZ = torch.empty((1, K, T, F), dtype=torch.float32, device=dev)
    MW = torch.empty_like(MZ)
    use_osn = "use_oracle_" in mask_for_z
    keep = {}
    # ---- step 1 per channel count
    for C, nodes in sorted(groups.items()):
        yd, sd, nd = _to_dev(y, nodes, dev), _to_dev(s, nodes, dev), _to_dev(n, nodes, dev)
        S, N = ops.stft(sd, n_fft), ops.stft(nd, n_fft)
        idx = torch.tensor(nodes, device=dev)
        Sref[0, idx], Nref[0, idx] = S[0, :, 0], N[0, :, 0]

        def om(kind):
            if kind == "ivad":
                return _ivad_mask(sd[:, :, 0], n_fft)
            return ops.tf_mask(_ref_plane(S, 0), _ref_plane(N, 0), kind)
        if masks is not None:
            mz = to_mask(masks[0], nodes)
        elif "rnn" in vads[0]:
            Yr = ops.stft(yd[:, :, 0].contiguous(), n_fft)
            mz = torch.stack([dnn_mask.estimate_mask(mods[0], spec_ft(Yr[0, i]), None, **dkw)
                              for i in range(len(nodes))])[None]
        else:
            mz = om(vads[0])
        st1 = tango_step1(yd, mz, n_fft, mu, filter_type, rank, 0, oracle_sn=(S, N) if use_osn else None)
        zs = ops.filter_sum(st1["W1"], S, None, conj=True, n_fft=n_fft)
        zn_ = ops.filter_sum(st1["W1"], N, None, conj=True, n_fft=n_fft)
        Z[0, idx], Zs[0, idx], Zn_[0, idx], ZN[0, idx] = st1["z_y"][0], zs[0], zn_[0], st1["zn"][0]
        Yref[0, idx] = st1["Y"][0, :, 0]
        MZ[0, idx] = mz[0]
        keep[C] = (nodes, st1["Y"], S, N, om)
    # ---- step-2 masks (tango.py:387-394)
    for C, (nodes, Y, S, N, om) in sorted(keep.items()):
        idx = torch.tensor(nodes, device=dev)
        if masks is not None:
            MW[0, idx] = to_mask(masks[1], nodes)[0]
        elif "rnn" in vads[1]:
            if mods[1] is None:
                MW[0, idx] = MZ[0, idx]
            else:
                for k in nodes:
                    others = [j for j in range(K) if j != k]
                    if z_sigs in ("zs_hat", "zn_hat"):
                        zin = Z if z_sigs == "zs_hat" else ZN
                        zl = [spec_ft(zin[0, j]) for j in others]
                    else:
                        zl = [spec_ft(t[0, j]) for j in others for t in (Z, ZN)]
                    MW[0, k] = dnn_mask.estimate_mask(mods[1], spec_ft(Yref[0, k]), zl, **dkw)
        else:
            MW[0, idx] = (MZ[0, idx] if vads[1] == vads[0] else om(vads[1])[0])
    # ---- what the other nodes contribute to the step-2 statistics (tango.py:396-429)
    z_rs = z_rn = None
    if mask_for_z == "distant":
        z_rs, z_rn = ops.apply_mask(Z, MW, False), ops.apply_mask(Z, MW, True)
    elif mask_for_z == "compressed":
        mc = ops.tf_mask(Zs, Zn_, vads[0])
        z_rs, z_rn = ops.apply_mask(Z, mc, False), ops.apply_mask(Z, mc, True)
    elif mask_for_z == "use_oracle_refs":
        z_rs, z_rn = Sref, Nref
    elif mask_for_z == "use_oracle_zs":
        z_rs, z_rn = Zs, Zn_
    elif mask_for_z != "local":              # 'previous' and any other string: unmasked z in both statistics
        z_rs = z_rn = Z
    # ---- step 2 per channel count
    res = {nm: np.empty((K, F, T), np.complex64) for nm in ("yf", "sf", "nf")}
    for C, (nodes, Y, S, N, om) in sorted(keep.items()):
        idx = torch.tensor(nodes, device=dev)
        mw = MW[:, idx].contiguous()
        yf, W2 = tango_step2(Y, Z, mw, n_fft, mu, filter_type, rank, "FT", node_sel=nodes, z_rs=z_rs, z_rn=z_rn)
        sf = ops.filter_sum(W2, S, Zs, conj=True, n_fft=n_fft, out_layout="FT", node_sel=nodes)
        nf = ops.filter_sum(W2, N, Zn_, conj=True, n_fft=n_fft, out_layout="FT", node_sel=nodes)
        for i, k in enumerate(nodes):
            res["yf"][k], res["sf"][k], res["nf"][k] = yf[0, i].cpu().numpy(), sf[0, i].cpu().numpy(), \
                nf[0, i].cpu().numpy()
    tr = lambda a: ops.transpose_last2(a)[0].cpu().numpy()
    res.update(z_y=tr(Z), z_s=tr(Zs), z_n=tr(Zn_), zn=tr(ZN), masks_z=tr(MZ), mask_w=tr(MW))
    return res
