"""Names of disco_theque/speech_enhancement/tango.py (:28-36, :41-139, :142-240, :252-457, :460-641)."""
import numpy as np

from ..evaluate import get_dset, get_directory_name, get_input_signals, load_models, main  # noqa: F401  (tango.py:41-139, 460)
from ..tango import offline_tango  # noqa: F401  (reference signature, tango.py:252)
from ._util import DEVICE
from .sigproc_utils import tf_mask, vad_oracle_batch

N_FFT = 512          # tango.py:28
N_HOP = 256          # tango.py:29
WIN_LEN = 21         # tango.py:34
PRED_FRAME = "mid"   # tango.py:35
MASK_Z = "local"     # tango.py:36


def concatenate_signals(y, z, k, m=1):
    """tango.py:142-155: own microphones of node k, then m * z of the other nodes in node order.
    Host-side helper (pure indexing); the kernels use the same channel order without materialising it."""
    z = np.array(z)
    return np.concatenate((y[k], m * z[:k], m * z[k + 1:]), axis=0)


def get_z_for_mask(z_s, z_n, k, nb_nodes=4, z_sigs="zs_hat"):
    """tango.py:158-186: which compressed signals feed the mask estimator of node k."""
    if z_sigs in ("zs_hat", "zn_hat"):
        z_in = z_s if z_sigs == "zs_hat" else z_n
        keep = [j for j in range(nb_nodes) if j != k]
        return np.array(z_in)[keep, :, :]
    z_in = np.concatenate((z_s, z_n), axis=0)
    z_out = 1 * z_in
    for i in range(z_in.shape[0]):                       # interleave zs_0, zn_0, zs_1, zn_1, ...
        z_out[i] = z_in[i // 2] if i % 2 == 0 else z_in[int(0.5 * (z_in.shape[0] - 1 + i))]
    keep = [c for c in range(2 * nb_nodes) if c not in (2 * k, 2 * k + 1)]
    return z_out[keep, :, :]


def reshape_mask(mask, output_frame="last"):
    """tango.py:228-240: (T, win, F) network output -> (F, T) mask."""
    if output_frame == "last":
        out = mask[:, -1, :]
    elif output_frame == "mid":
        w = np.shape(mask)[1]
        out = mask[:, int(np.floor(w / 2)):int(np.ceil(w / 2)), :]
    elif output_frame == "all":
        raise NotImplementedError("This case was not implemented yet")
    else:
        raise ValueError(":param output_frame: should be either 'last', 'all' or 'mid'")
    return np.squeeze(out).T


def get_mask(y, ss, sn, sz=None, mask_type="irm1", mod=None, ts=None, **kwargs):
    """tango.py:189-225: oracle masks ('irmX' / 'ibmX' / 'iamX' / 'ivad') or the mask a network predicts
    ('crnn' / 'rnn': `mod` on the device through disco_b200.dnn_mask, window keywords win_len / win_hop /
    frame_to_pred as in the reference).  Returns an (F, T) array like the reference."""
    if mask_type[:-1] in ("irm", "ibm", "iam"):
        return tf_mask(ss, sn, type=mask_type)
    if "rnn" in mask_type:                                   # tango.py:209-215
        from .. import dnn_mask
        if mask_type != "crnn":
            raise NotImplementedError("only the 3-D ('crnn') input arrangement of prepare_data is implemented")
        kw = {k: kwargs[k] for k in ("win_len", "win_hop", "frame_to_pred", "norm_type") if k in kwargs}
        m = dnn_mask.estimate_mask(mod, y, sz, device=DEVICE, **kw)            # (T, F) on the device
        return m.T.cpu().numpy()
    if mask_type == "ivad":
        m = np.zeros(np.shape(ss))
        vad = vad_oracle_batch(ts, win_len=N_FFT, win_hop=N_HOP)[::N_HOP]
        m[:, :len(vad)] = np.tile(vad, (np.shape(ss)[0], 1))
        return m
    raise ValueError("Unknown value for `mask_type`")
