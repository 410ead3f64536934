"""Step-1 driver: the reference's get_z_signals.main (disco_theque/speech_enhancement/get_z_signals.py:320-404) over a
range of RIRs, in batched device calls.

Per RIR the reference reads 48 convolved WAVs (get_input_signals, :44-92), runs step 1 of Tango with one mask type
(offline_tango, :213-317) and saves, per node, the compressed signal z_y ('zs_hat') and zn = Y_ref - z_y ('zn_hat'),
raw complex64 and their magnitudes, under <dataset>/disco/<scenario>/<dset>/stft_z/<save_dir>/: the inputs the
step-2 CRNN is trained on.  `main` does the same for RIRs i_rir .. i_rir + nb_rir - 1, `batch` of them per device
call: they are zero-padded to the longest and passed with their own lengths to

    step-1 masks (tango._step1_mask)  ->  tango.tango_step1

one call each, then one device-to-host copy of z_y and zn.  A reader thread reads batch i + 1 and a writer thread
writes batch i - 1 (dataset_post.save_z_signals, which takes the magnitudes with NumPy as the reference does) while the
device works on batch i.

    python -m disco_b200.get_z -vt irm1 -sd out --rir 11001 --nb_rir 1000 --dataset ../dataset

Deviations from the reference, each a fix of one of its bugs:
  * main calls load_models(vad_type, weights) (:343), which takes one argument (:95), so the reference raises
    TypeError for every mask type.  Here weights_sc is loaded when, and only when, vad_type names a network
    ('crnn' / 'rnn'); a network without weights_sc raises ValueError.  The command line's default -msc './' (a
    directory) is therefore harmless with oracle masks.
  * its "already processed" test (:328-331) looks for the last file without the '.npy' np.save appends, so it never
    matches and every run recomputes everything.  Here an RIR is skipped, with the reference's message, when that
    file exists; an RIR with only some of its files is redone.
"""
import argparse
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import ops
from .dataset_post import save_z_signals
from .evaluate import _read_convolved, _to_host, get_directory_name, get_dset
from .evaluate import load_models as _load_models
from .tango import _frame_clip, _mask_kind, _ref_plane, _step1_mask, _uneven_lengths, tango_step1

N_FFT = 512                  # get_z_signals.py:17
MASK_Z = "local"             # get_z_signals.py:25
SNR_RANGE = [[0, 6]]         # get_z_signals.py:26
PATH_TO_DATASET = "../../../dataset"      # get_z_signals.py:27


def get_input_signals(i_rir, scenario="living", noise="ssn", snr_range=None, *, path_to_dataset=PATH_TO_DATASET,
                      nb_ch=(4, 4, 4, 4)):
    """get_z_signals.py:44-92: the convolved mixture, target and noise of every microphone of RIR i_rir, lists
    [node][ch] of float32 arrays.  Every file must have the length and rate of the first: ValueError naming the file
    otherwise; a missing file raises FileNotFoundError with its path."""
    path_to_set = os.path.join(path_to_dataset, "disco", scenario, get_dset(i_rir))
    dirry = get_directory_name([[0, 6]] if snr_range is None else snr_range)
    y, s, n, _ = _read_convolved(os.path.join(path_to_set, "wav_processed", dirry, ""), i_rir, noise, nb_ch)
    return y, s, n


def load_models(weightss, *, device=None):
    """get_z_signals.py:95-120: [the single-channel reference CRNN with the weights of checkpoint weightss[0] (its
    'model_state_dict'), or None], put on `device` (default: CUDA) in evaluation mode."""
    return _load_models([None], list(weightss[:1]), [1], device=device)


def _save_root(path_to_dataset, scenario, rir, save_dir):
    return os.path.join(path_to_dataset, "disco", scenario, get_dset(rir), "stft_z", save_dir, "")


def _batch_plan(i_rir, nb_rir, batch, noise, scenario, save_dir, path_to_dataset, nb_nodes):
    """The RIRs still to do, in RIR order, cut into batches of up to `batch`.  An RIR whose last file,
    normed/abs/<snr>/zn_hat/<rir>_<noise>_Node-<nb_nodes>.npy, exists is skipped with the reference's message
    (get_z_signals.py:328-331, which omits the '.npy' and so never skips)."""
    dirry = get_directory_name(SNR_RANGE)
    todo = []
    for rir in range(i_rir, i_rir + nb_rir):
        last = os.path.join(_save_root(path_to_dataset, scenario, rir, save_dir), "normed", "abs", dirry, "zn_hat",
                            "{}_{}_Node-{}.npy".format(str(rir), noise, str(nb_nodes)))
        if os.path.isfile(last):
            print("Conf {} with {} noise already processed".format(str(rir), noise))
            continue
        todo.append(rir)
    step = max(1, int(batch))
    return [todo[i:i + step] for i in range(0, len(todo), step)]


def _read_batch(rirs, scenario, noise, path_to_dataset, nb_ch):
    """Host half of a batch: every RIR's y, s, n zero-padded to the batch's longest and stacked, [3, B, K, C, L_max]
    float32, and their lengths."""
    items = [get_input_signals(rir, scenario, noise, SNR_RANGE, path_to_dataset=path_to_dataset, nb_ch=nb_ch)
             for rir in rirs]
    lengths = np.array([len(it[0][0][0]) for it in items], dtype=np.int64)
    sig = np.zeros((3, len(rirs), len(nb_ch), nb_ch[0], int(lengths.max())), dtype=np.float32)
    for b, it in enumerate(items):
        for i in range(3):
            sig[i, b, :, :, :lengths[b]] = np.asarray(it[i])
    return {"rirs": list(rirs), "sig": sig, "lengths": lengths}


def _network_masks(vad, mods, y, lengths):
    """Step-1 masks [B, K, T, F] of the network mods[0] (vad 'crnn' / 'rnn'), each RIR's computed on its own frames
    from the spectrum of its reference microphones alone, as compat.get_z_signals.offline_tango computes them, and 0
    past them.  The network must see a lone RIR's input: prepare_data clamps |Y| to at least 1e-6 before zero-padding
    the window edges, so the last windows of a padded RIR would see clamped 1e-6 frames instead of zeros."""
    B, K, _, L = y.shape
    mask = torch.zeros((B, K, ops.n_frames(L, N_FFT), N_FFT // 2 + 1), dtype=torch.float32, device=y.device)
    for b, Lb in enumerate(int(v) for v in lengths):
        y0 = y[b:b + 1, :, 0, :Lb].contiguous()
        mask[b, :, :ops.n_frames(Lb, N_FFT)] = _step1_mask(vad, mods, None, None, lambda: ops.stft(y0, N_FFT),
                                                           N_FFT)[0]
    return mask


def _compress(data, vad, mods, mask_for_z, dev):
    """Device half of a batch: the step-1 masks of vad and one tango_step1 call.  Returns z_y and zn [B, K, T, F]
    complex64 device tensors.  'use_oracle_*' mask_for_z takes the statistics of the clean spectra
    (get_z_signals.py:282-284); every other value the masked mixture (:285-287)."""
    sig, lengths = data["sig"], data["lengths"]
    y = torch.from_numpy(sig[0]).to(dev)
    B, K, C, L = y.shape
    lens = _uneven_lengths(lengths, B, L, N_FFT)
    stft = (lambda a: ops.stft(a, N_FFT)) if lens is None else (lambda a: ops.stft_lengths(a, lens, N_FFT))
    osn = None
    if "use_oracle_" in mask_for_z:
        s, n = (torch.from_numpy(sig[i]).to(dev) for i in (1, 2))
        S, N = osn = stft(s), stft(n)
    if _mask_kind(vad) == "dnn":
        mask = _network_masks(vad, mods, y, lengths)
    else:
        if osn is not None:
            spectra, s0 = (lambda: (_ref_plane(S, 0), _ref_plane(N, 0))), s[:, :, 0]
        else:
            # only the reference microphones' clean signals are needed
            s0, n0 = (torch.from_numpy(np.ascontiguousarray(sig[i][:, :, 0])).to(dev) for i in (1, 2))
            spectra = lambda: (stft(s0), stft(n0))
        mask = _step1_mask(vad, None, spectra, s0, None, N_FFT, lens)
    if lens is not None:
        # past an RIR's end its spectra are 0 and an oracle mask 0/0
        mask = _frame_clip(lens, ops.n_frames(L, N_FFT), N_FFT, dev)(mask)
    st1 = tango_step1(y, mask, N_FFT, oracle_sn=osn, lengths=lens)
    return {"z_y": st1["z_y"], "zn": st1["zn"]}


def _write_batch(data, res, save_dir, noise, scenario, path_to_dataset):
    """Files of every RIR of a batch (get_z_signals.py:350-360): per node (F, T_b) complex64 zs_hat / zn_hat, cut to
    the RIR's own T_b = 1 + L_b // hop frames, and their magnitudes."""
    dirry = get_directory_name(SNR_RANGE)
    for b, rir in enumerate(data["rirs"]):
        Tb = ops.n_frames(int(data["lengths"][b]), N_FFT)
        ft = lambda a: [np.ascontiguousarray(a[b, k, :Tb].T) for k in range(a.shape[1])]
        save_z_signals(ft(res["z_y"]), ft(res["zn"]), _save_root(path_to_dataset, scenario, rir, save_dir), dirry,
                       rir, noise)
        print(str(rir) + "  done")


def main(vad_type, save_dir, i_rir, noise, scenario="living", mask_z=MASK_Z, weights_sc=None, *, nb_rir=1, batch=8,
         path_to_dataset=PATH_TO_DATASET, nb_ch=(4, 4, 4, 4), device=None):
    """get_z_signals.main (get_z_signals.py:320-360) for RIRs i_rir .. i_rir + nb_rir - 1, up to `batch` RIRs per
    device call.

    The positional parameters are the reference's.  vad_type is one mask type: 'irmX' / 'ibmX' / 'iamX', 'ivad', or
    'crnn' / 'rnn' (the single-channel CRNN of checkpoint weights_sc, predicting the middle frame of 21).  Keyword-only:
    nb_rir, batch; path_to_dataset, nb_ch (module globals in the reference); device (default CUDA).  Files are written
    under <path_to_dataset>/disco/<scenario>/<dset>/stft_z/<save_dir>/ with the reference's names.  RIRs whose last
    file exists are skipped before their files are read.  The argument errors (mask_z None: TypeError, as the
    reference's; an unknown vad_type, a network without weights_sc, uneven nb_ch: ValueError) are raised before any
    file is read."""
    if mask_z is None:
        raise TypeError("argument of type 'NoneType' is not iterable")   # reference get_z_signals.py:282
    kind = _mask_kind(vad_type)
    if kind == "dnn" and weights_sc is None:
        raise ValueError("vad_type=%r predicts the masks with a network: weights_sc must name its checkpoint"
                         % (vad_type,))
    if len(set(nb_ch)) != 1:
        raise ValueError("every node must have the same number of microphones, got nb_ch=%s" % (list(nb_ch),))
    dev = torch.device("cuda" if device is None else device)
    mods = load_models([weights_sc], device=dev) if kind == "dnn" else [None]
    plan = _batch_plan(i_rir, nb_rir, batch, noise, scenario, save_dir, path_to_dataset, len(nb_ch))
    if not plan:
        return
    read = lambda rirs: _read_batch(rirs, scenario, noise, path_to_dataset, nb_ch)
    write = lambda data, res: _write_batch(data, res, save_dir, noise, scenario, path_to_dataset)
    with ThreadPoolExecutor(max_workers=1) as reader, ThreadPoolExecutor(max_workers=1) as writer:
        nxt, wrote = reader.submit(read, plan[0]), None
        for i in range(len(plan)):
            data = nxt.result()
            if i + 1 < len(plan):
                nxt = reader.submit(read, plan[i + 1])
            res = _to_host(_compress(data, vad_type, mods, mask_z, dev))
            if wrote is not None:
                wrote.result()                 # one batch in writing at a time; its error surfaces here
            wrote = writer.submit(write, data, res)
        wrote.result()


def _parser():
    """The reference's flags (get_z_signals.py:365-392) and this driver's additions."""
    p = argparse.ArgumentParser(description="DONSE arguments")
    p.add_argument("--vad_type", "-vt", type=str, default="irm1")
    p.add_argument("--sav_dir", "-sd", type=str, help="Dir to save results under")
    p.add_argument("--rir", type=int, help="RIR of signal to filter")
    p.add_argument("--scenario", "-scene", type=str, help="Scenario to use", choices=["living", "meeting", "random"],
                   default="living")
    p.add_argument("--noise", type=str, choices=["ssn", "it", "fs"], default="fs")
    p.add_argument("--mask_z", "-mz", type=str, help="Mask to apply on z",
                   choices=["None", "local", "distant", "compressed", "use_oracle_refs", "use_oracle_zs"],
                   default="local")
    p.add_argument("--mod_sc", "-msc", type=str, help="Name of single-channel model", default="./")
    p.add_argument("--nb_rir", type=int, default=1, help="number of consecutive RIRs from --rir on")
    p.add_argument("--batch", type=int, default=8, help="RIRs per device call")
    p.add_argument("--dataset", type=str, default=PATH_TO_DATASET, help="root of the data set (holds disco/)")
    return p


def parse_args(argv=None):
    """Command line -> (positional arguments, keyword arguments) of main, converted as get_z_signals.py:394-404
    does."""
    a = _parser().parse_args(argv)
    return ((a.vad_type, a.sav_dir, a.rir, a.noise),
            dict(scenario=a.scenario, mask_z=None if a.mask_z == "None" else a.mask_z,
                 weights_sc=None if a.mod_sc == "None" else a.mod_sc, nb_rir=a.nb_rir, batch=a.batch,
                 path_to_dataset=a.dataset))


if __name__ == "__main__":
    args, kwargs = parse_args()
    main(*args, **kwargs)
