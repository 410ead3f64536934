"""Step-1-only variant of Tango (disco_theque/speech_enhancement/get_z_signals.py:213-317): produces the
compressed signals that are saved as DNN training inputs (get_z_signals.py:350-359).  main and its helpers
(get_z_signals.py:30-120, 320-360) are those of the batched driver, disco_b200.get_z."""
import torch

from .. import ops
from ..get_z import get_dset, get_directory_name, get_input_signals, load_models, main  # noqa: F401  (:30-120, 320)
from ..tango import _ref_plane, _reference_lists, _step1_mask, _to_dev, tango_step1


def offline_tango(y, s, n, vads="irm1", mods=None, mask_for_z="local", *, n_fft=512, mu=1, filter_type="gevd",
                  rank=1, device="cuda"):
    """Reference signature.  y, s, n: [node][channel] 1-D float32 signals (equal channel counts).
    `vads` is ONE mask type here (get_z_signals.py:279).  Returns the reference's 5 lists (length K) of
    (F, T) arrays: z_y, z_s, z_n, zn (complex64), masks_z."""
    vad = vads if isinstance(vads, str) else vads[0]
    if len({len(c) for c in y}) != 1:
        raise NotImplementedError("ragged channel counts: use disco_b200.tango.offline_tango")
    dev = torch.device(device)
    nodes = list(range(len(y)))
    yd, sd, nd = _to_dev(y, nodes, dev), _to_dev(s, nodes, dev), _to_dev(n, nodes, dev)
    S, N = ops.stft(sd, n_fft), ops.stft(nd, n_fft)
    mask_z = _step1_mask(vad, mods, lambda: (_ref_plane(S, 0), _ref_plane(N, 0)), sd[:, :, 0],
                         lambda: ops.stft(yd[:, :, 0].contiguous(), n_fft), n_fft)
    osn = (S, N) if (mask_for_z is not None and "use_oracle_" in mask_for_z) else None
    st1 = tango_step1(yd, mask_z, n_fft, mu, filter_type, rank, 0, oracle_sn=osn)
    z_s = ops.filter_sum(st1["W1"], S, None, conj=True, n_fft=n_fft)
    z_n = ops.filter_sum(st1["W1"], N, None, conj=True, n_fft=n_fft)
    to_ft = lambda a: ops.transpose_last2(a)[0].cpu().numpy()
    res = dict(z_y=to_ft(st1["z_y"]), z_s=to_ft(z_s), z_n=to_ft(z_n), zn=to_ft(st1["zn"]), masks_z=to_ft(mask_z))
    return _reference_lists(res, ("z_y", "z_s", "z_n", "zn", "masks_z"), [vad, vad])
