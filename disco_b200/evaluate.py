"""Evaluation driver: the reference's tango.main (disco_theque/speech_enhancement/tango.py:460-641) over a range of
RIRs, in batched device calls.

Per RIR the reference reads 48 convolved WAVs, 2 dry sources and the mixing SNR (get_input_signals, :55-111),
beamforms, converts the six outputs back to time signals, scores them (BSS-eval, STOI, fw_snr, fw_sd) and writes
WAV/, MASK/, STFT/z/raw/ and the two OIM/results_{tango,mwf}_<rir>_<noise>.p pickles under
results/<scenario>/<dset>/<save_dir>/.  `main` does the same for RIRs i_rir .. i_rir + nb_rir - 1, `batch` of them
per device call: they are zero-padded to the longest and passed with their own lengths to

    tango_batched (or online.online_tango)  ->  post.to_time  ->  post.tango_scores(stoi=True)

one call each, then one device-to-host copy of everything the files need.  A background thread reads the next
batch's WAVs while the device works on the current one.  Files, names and pickle keys are the reference's; RIRs whose
results_mwf pickle exists are skipped, as the reference skips them.

    python -m disco_b200.evaluate -vt irm1 irm1 -sd out --rir 11001 --nb_rir 1000 --dataset ../dataset

Not ported: save_conf (:243-249), the matplotlib figure of the room set-up.  FIG/ is created, as the reference
creates it, and stays empty.
"""
import argparse
import os
import pickle
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import ops, post, wav_io
from .online import online_tango
from .tango import _mask_kind, _step1_mask, _step2_mask, tango_batched

N_FFT = 512                  # tango.py:28
MASK_Z = "local"             # tango.py:36
SNR_RANGE = [[0, 6]]         # tango.py:37
PATH_TO_DATASET = "../../../dataset"      # tango.py:38

# keys of the two result pickles in the reference's order (tango.py:617-632); 'snr_in_raw' is the loaded SNR
RESULTS_TANGO = ("snr_in_raw", "sar_cnv", "sir_cnv", "sdr_cnv", "delta_stoi_cnv", "delta_stoi_dry", "snr_out",
                 "snr_in_cnv", "snr_in_dry", "fw_sd_cnv", "fw_sd_dry", "sar_dry", "sir_dry", "sdr_dry", "sdr_in_cnv",
                 "sir_in_cnv", "sdr_in_dry", "sir_in_dry", "sar_in_dry")
RESULTS_MWF = tuple("delta_stoi" if k == "delta_stoi_cnv" else k for k in RESULTS_TANGO)
# WAV name -> (time signal of to_time, or None for the input at the reference microphone; input array)
_WAVS = (("in_mix", None, "y"), ("out_mix", "yf", None), ("mid_z", "z_y", None), ("in_noi", None, "n"),
         ("out_noi", "nf", None), ("in_tar", None, "s"), ("out_tar", "sf", None))


def get_dset(rir):
    """Given  `rir`, return 'test' or 'train' corresponding to dataset (tango.py:41-45)."""
    assert 0 < rir < 12001, "rir ID should be between 1 and 12000"
    return "train" if rir < 11001 else "test"


def get_directory_name(snr_range):
    """From `snr_range`, return the name of the directory in form of e.g. 0-6 or 3-6_5-15 (tango.py:48-52)."""
    return "_".join(["{}-{}".format(str(snr_range[k][0]), str(snr_range[k][1])) for k in range(len(snr_range))])


def _read(path):
    """wav_io.read of a float32 signal -> (x, fs), or FileNotFoundError naming the path."""
    if not os.path.isfile(path):
        raise FileNotFoundError("no such file: %s" % path)
    return wav_io.read(path, dtype="float32")


def _read_convolved(root, i_rir, noise, nb_ch):
    """The convolved target, noise and mixture of every microphone of RIR i_rir under wav_processed/<snr>/ (`root`),
    as tango.py:74-109 and get_z_signals.py:75-90 read them: lists [node][ch] of float32 arrays, and their rate.
    Every file must have the length and rate of the first: ValueError naming the file otherwise; a missing file
    raises FileNotFoundError with its path."""
    y, s, n = ([[] for _ in nb_ch] for _ in range(3))
    fs = length = None
    ii_ch = 0
    for i_nod in range(len(nb_ch)):
        for _ in range(nb_ch[i_nod]):
            ii_ch += 1
            for lst, path in ((s, root + "target/{}_Ch-{}.wav".format(i_rir, ii_ch)),
                              (n, root + "noise/{}_{}_Ch-{}.wav".format(i_rir, noise, ii_ch)),
                              (y, root + "mixture/{}_{}_Ch-{}.wav".format(i_rir, noise, ii_ch))):
                x, rate = _read(path)
                if fs is None:
                    fs, length = rate, len(x)
                if rate != fs or len(x) != length:
                    raise ValueError("%s: %d samples at %d Hz, the RIR's first file has %d at %d Hz"
                                     % (path, len(x), rate, length, fs))
                lst[i_nod].append(x)
    return y, s, n, fs


def get_input_signals(i_rir, scenario="living", noise="ssn", snr_range=None, *, path_to_dataset=PATH_TO_DATASET,
                      nb_ch=(4, 4, 4, 4)):
    """tango.py:55-111: the convolved target, noise and mixture of every microphone of RIR i_rir (lists [node][ch]
    of float32 arrays), the dry target and noise, the sampling rate and the mixing SNR stored with the data set.
    n_dry is scaled by that SNR in float32, as the reference's in-place `*=` on its float32 array does.
    Every convolved file must have the length and rate of the first and the dry files its rate: ValueError naming
    the file otherwise; a missing file raises FileNotFoundError with its path."""
    path_to_set = os.path.join(path_to_dataset, "disco", scenario, get_dset(i_rir))
    dirry = get_directory_name([[0, 6]] if snr_range is None else snr_range)
    snr_file = os.path.join(path_to_set, "log", "snrs", "dry", dirry, "") + "{}_{}.npy".format(str(i_rir), noise)
    if not os.path.isfile(snr_file):
        raise FileNotFoundError("no such file: %s" % snr_file)
    snrs_used = np.load(snr_file, allow_pickle=True)[0]
    y, s, n, fs = _read_convolved(os.path.join(path_to_set, "wav_processed", dirry, ""), i_rir, noise, nb_ch)
    dry = []
    for path in (os.path.join(path_to_set, "wav_original/dry/target/") + str(i_rir) + "_S-1.wav",
                 os.path.join(path_to_set, "wav_original/dry/noise/") + str(i_rir) + "_S-2_" + noise + ".wav"):
        x, rate = _read(path)
        if rate != fs:
            raise ValueError("%s: %d Hz, the RIR's convolved files have %d Hz" % (path, rate, fs))
        dry.append(x)
    s_dry, n_dry = dry
    n_dry *= np.float32(10 ** (-snrs_used / 20))
    return y, s, n, s_dry, n_dry, fs, snrs_used


def load_models(types, models, nodes_nbs, *, device=None):
    """tango.py:114-139: for each step, the reference CRNN with nodes_nbs[step] input channels and the weights of
    checkpoint models[step] (its 'model_state_dict'; the keys are the reference's), or None.  The models are put on
    `device` (default: CUDA) in evaluation mode."""
    from . import dnn_mask
    device = torch.device("cuda" if device is None else device)
    out = []
    for i_step in range(len(types)):
        if models[i_step] is None:
            out.append(None)
            continue
        model = dnn_mask.build_crnn(int(nodes_nbs[i_step]))
        saved = torch.load(models[i_step], map_location="cpu")
        model.load_state_dict(saved["model_state_dict"])
        out.append(model.to(device).eval())
    return out


def _results_dir(results_root, scenario, rir, save_dir):
    return os.path.join(results_root, scenario, get_dset(rir), save_dir, "")


def _batch_plan(i_rir, nb_rir, batch, noise, scenario, save_dir, results_root):
    """The RIRs still to do, in RIR order, cut into batches of up to `batch`.  An RIR whose results_mwf pickle exists
    is skipped with the reference's message (tango.py:477-479); one with only results_tango is redone."""
    todo = []
    for rir in range(i_rir, i_rir + nb_rir):
        if os.path.isfile(_results_dir(results_root, scenario, rir, save_dir) + "OIM/results_mwf_" + str(rir) + "_"
                          + noise + ".p"):
            print("Conf {} with {} noise already processed".format(str(rir), noise))
            continue
        todo.append(rir)
    step = max(1, int(batch))
    return [todo[i:i + step] for i in range(0, len(todo), step)]


def _read_batch(rirs, scenario, noise, path_to_dataset, nb_ch):
    """Host half of a batch: every RIR's signals zero-padded to the batch's longest and stacked, y, s, n
    [B, K, C, L_max], s_dry, n_dry [B, L_dry_max] float32, their lengths and the common rate."""
    items = [get_input_signals(rir, scenario, noise, SNR_RANGE, path_to_dataset=path_to_dataset, nb_ch=nb_ch)
             for rir in rirs]
    fs = items[0][5]
    for rir, it in zip(rirs, items):
        if it[5] != fs:
            raise ValueError("RIR %d: %s is at %d Hz, RIR %d of the same batch at %d Hz"
                             % (rir, _first_file(rir, scenario, noise, path_to_dataset), it[5], rirs[0], fs))
    lengths = np.array([len(it[0][0][0]) for it in items], dtype=np.int64)
    d_len = [(len(it[3]), len(it[4])) for it in items]
    B, K, C, L = len(rirs), len(nb_ch), nb_ch[0], int(lengths.max())
    sig = np.zeros((3, B, K, C, L), dtype=np.float32)
    dry = np.zeros((2, B, max(max(d) for d in d_len)), dtype=np.float32)
    for b, it in enumerate(items):
        for i in range(3):
            sig[i, b, :, :, :lengths[b]] = np.asarray(it[i])
        dry[0, b, :d_len[b][0]], dry[1, b, :d_len[b][1]] = it[3], it[4]
    score_len = np.array([min(lengths[b], *d_len[b]) for b in range(B)], dtype=np.int64)
    return {"rirs": list(rirs), "sig": sig, "dry": dry, "lengths": lengths, "score_len": score_len, "fs": fs,
            "snrs": [it[6] for it in items]}


def _first_file(rir, scenario, noise, path_to_dataset):
    dirry = get_directory_name(SNR_RANGE)
    return os.path.join(path_to_dataset, "disco", scenario, get_dset(rir), "wav_processed", dirry, "target",
                        "{}_Ch-1.wav".format(rir))


def _network_masks(vads, mods, z_sigs, y, s, n, lengths, n_fft):
    """(mask_z [B, K, T, F], callable mask_w) of network masks for tango_batched, each RIR's computed on its own
    frames by the helpers offline_tango uses, and 0 past them.  The network must see a lone RIR's input: prepare_data
    clamps |Y| to at least 1e-6 and then zero-pads the window edges, so the last windows of a padded RIR would see
    clamped 1e-6 frames instead of zeros."""
    B, K, _, L = y.shape
    T, F = ops.n_frames(L, n_fft), n_fft // 2 + 1
    frames = [ops.n_frames(int(Lb), n_fft) for Lb in lengths]
    lone = [tuple(x[b:b + 1, ..., :Lb] for x in (y, s, n)) for b, Lb in enumerate(lengths)]
    stft0 = lambda x: ops.stft(x[:, :, 0].contiguous(), n_fft)          # microphone 0 alone, as offline_tango
    mask_z = torch.zeros((B, K, T, F), dtype=torch.float32, device=y.device)
    for b, (yb, sb, nb) in enumerate(lone):
        mask_z[b, :, :frames[b]] = _step1_mask(vads[0], mods, lambda: (stft0(sb), stft0(nb)), sb[:, :, 0],
                                               lambda: stft0(yb), n_fft)[0]

    def mask_w(Y, z_y, zn):
        out = torch.zeros_like(mask_z)
        for b, (yb, sb, nb) in enumerate(lone):
            t = frames[b]
            out[b, :, :t] = _step2_mask(vads, mods, mask_z[b:b + 1, :, :t], lambda: (stft0(sb), stft0(nb)),
                                        sb[:, :, 0], n_fft, Y[b:b + 1, :, 0, :t],
                                        (z_y[b:b + 1, :, :t], zn[b:b + 1, :, :t]), z_sigs=z_sigs)[0]
        return out
    return mask_z, mask_w


def _beamform(data, vads, mods, mask_z, z_sigs, online, block, lag, lambda_cor, dev):
    """Device half of a batch: beamforming, time signals and scores.  Returns the flat dict of device tensors the
    files need."""
    sig = torch.from_numpy(data["sig"]).to(dev)
    y, s, n = sig[0], sig[1], sig[2]
    s_dry, n_dry = (t for t in torch.from_numpy(data["dry"]).to(dev))
    lengths, fs = data["lengths"], data["fs"]
    L = y.shape[-1]
    if online:
        out = online_tango(y, s=s, n=n, vads=vads, mask_for_z=mask_z, block=block, lag=lag, lambda_cor=lambda_cor,
                           lengths=lengths)
    else:
        masks = None
        if "dnn" in [_mask_kind(v) for v in vads]:
            masks = _network_masks(vads, mods, z_sigs, y, s, n, lengths, N_FFT)
        out = tango_batched(y, s, n, masks=masks, vads=vads, mask_for_z=mask_z, lengths=lengths, out_layout="TF")
    times = post.to_time(out, L, layout="TF", lengths=lengths)
    results, resultsz = post.tango_scores(y[:, :, 0], s[:, :, 0], n[:, :, 0], s_dry, n_dry, times, fs, stoi=True,
                                          lengths=data["score_len"])
    flat = {"t_" + k: v for k, v in times.items()}
    flat.update(masks_z=out["masks_z"], mask_w=out["mask_w"], z_y=out["z_y"])
    flat.update({"tango_" + k: v for k, v in results.items()})
    flat.update({"mwf_" + k: v for k, v in resultsz.items()})
    return flat


def _to_host(tensors):
    """One device-to-host copy of a dict of device tensors (float32, float64 and complex64) -> dict of NumPy arrays."""
    names = list(tensors)
    parts = [tensors[k].contiguous().view(-1).view(torch.float32) for k in names]
    host = torch.cat(parts).cpu().numpy()
    out, pos = {}, 0
    for k, p in zip(names, parts):
        t = tensors[k]
        out[k] = host[pos:pos + p.numel()].view(str(t.dtype).replace("torch.", "")).reshape(tuple(t.shape))
        pos += p.numel()
    return out


def _mask_file_dtype(vad):
    """The dtype the reference's masks have on disk: bool for 'ibmX', float64 for 'ivad', float32 otherwise."""
    return bool if "ibm" in vad else (np.float64 if vad == "ivad" else np.float32)


def _write_batch(data, res, vads, save_dir, noise, scenario, results_root):
    """Files of every RIR of a batch, node by node, as tango.py:484-488 and :596-635 name them."""
    dirry = get_directory_name(SNR_RANGE)
    fs = data["fs"]
    j = os.path.join
    for b, rir in enumerate(data["rirs"]):
        root = _results_dir(results_root, scenario, rir, save_dir)
        for sub in (j("WAV", str(rir)), j("STFT", "z", "raw", dirry), "OIM", "FIG", j("MASK", str(rir))):
            os.makedirs(j(root, sub), exist_ok=True)
        Lb = int(data["lengths"][b])
        Tb = ops.n_frames(Lb, N_FFT)
        inputs = dict(zip("ysn", data["sig"][:, b, :, 0, :Lb]))              # reference microphone of every node
        K = inputs["y"].shape[0]
        for k in range(K):
            tag = "-" + noise + "_Node-" + str(k + 1)
            for name, t, x in _WAVS:
                wav = inputs[x][k] if t is None else res["t_" + t][b, k, :Lb]
                wav_io.write(root + "WAV/" + str(rir) + "/" + name + tag + ".wav", wav, fs)
            for step, key, vad in ((1, "masks_z", vads[0]), (2, "mask_w", vads[1])):
                m = np.ascontiguousarray(res[key][b, k, :Tb].T).astype(_mask_file_dtype(vad))
                np.save(root + "MASK/" + str(rir) + "/step" + str(step) + "_" + noise + "_Node-" + str(k + 1), m)
            np.save(j(root, "STFT", "z", "raw", dirry, "") + "{}_{}_Node-{}".format(str(rir), noise, str(k + 1)),
                    np.ascontiguousarray(res["z_y"][b, k, :Tb].T))
        for prefix, keys in (("tango", RESULTS_TANGO), ("mwf", RESULTS_MWF)):
            d = {k: data["snrs"][b] if k == "snr_in_raw" else np.array(res[prefix + "_" + k][b], dtype=np.float64)
                 for k in keys}
            with open(root + "OIM/results_" + prefix + "_" + str(rir) + "_" + noise + ".p", "wb") as fh:
                pickle.dump(d, fh)
        print(str(rir) + "  done")


def main(vad_types, save_dir, i_rir, noise, scenario="living", mask_z=MASK_Z, z_sigs="zs_hat", models=[None, None],
         *, nb_rir=1, batch=8, path_to_dataset=PATH_TO_DATASET, results_root="results", nb_ch=(4, 4, 4, 4),
         online=False, block=8, lag=1, lambda_cor=0.95, device=None):
    """tango.main (tango.py:460-641) for RIRs i_rir .. i_rir + nb_rir - 1, up to `batch` RIRs per device call.

    The positional parameters are the reference's.  Keyword-only: nb_rir, batch; path_to_dataset, nb_ch (module
    globals in the reference); results_root (the reference writes under ./results); online=True runs
    online.online_tango with block, lag and lambda_cor instead of the offline beamformer ('crnn' masks are not causal
    and raise ValueError there); device (default CUDA).  Files are written under
    <results_root>/<scenario>/<dset>/<save_dir>/ with the reference's names.  RIRs whose results_mwf pickle exists are
    skipped before their files are read.  The reference's room figure (save_conf) is not drawn."""
    vads = list(vad_types)
    kinds = [_mask_kind(v) for v in vads]
    if online and "dnn" in kinds:
        raise ValueError("online mode takes no network masks: the reference CRNN predicts the middle frame of a "
                         "21-frame window and is not causal")
    if len(set(nb_ch)) != 1:
        raise ValueError("every node must have the same number of microphones, got nb_ch=%s" % (list(nb_ch),))
    dev = torch.device("cuda" if device is None else device)
    K = len(nb_ch)
    nodes_nbs = [1, K] if z_sigs in ("zs_hat", "zn_hat") else [1, 1 + 2 * (K - 1)]      # tango.py:493
    mods = load_models(vads, models, nodes_nbs, device=dev)
    plan = _batch_plan(i_rir, nb_rir, batch, noise, scenario, save_dir, results_root)
    if not plan:
        return
    read = lambda rirs: _read_batch(rirs, scenario, noise, path_to_dataset, nb_ch)
    with ThreadPoolExecutor(max_workers=1) as pool:
        nxt = pool.submit(read, plan[0])
        for i in range(len(plan)):
            data = nxt.result()
            if i + 1 < len(plan):
                nxt = pool.submit(read, plan[i + 1])
            res = _to_host(_beamform(data, vads, mods, mask_z, z_sigs, online, block, lag, lambda_cor, dev))
            _write_batch(data, res, vads, save_dir, noise, scenario, results_root)


def _parser():
    """The reference's flags (tango.py:646-677) and this driver's additions."""
    p = argparse.ArgumentParser(description="DONSE arguments")
    p.add_argument("--vad_type", "-vt", type=str, nargs=2)
    p.add_argument("--sav_dir", "-sd", type=str, help="Dir to save results under")
    p.add_argument("--rir", type=int, help="RIR of signal to filter")
    p.add_argument("--scenario", "-scene", type=str, help="Scenario to use", choices=["living", "meeting", "random"],
                   default="living")
    p.add_argument("--noise", type=str, choices=["ssn", "it", "fs"], default="fs")
    p.add_argument("--mask_z", "-mz", type=str, help="Mask to apply on z",
                   choices=["None", "local", "distant", "compressed", "use_oracle_refs", "use_oracle_zs"],
                   default="local")
    p.add_argument("--mods", "-m", type=str, nargs=2, help="Name (path + name) of trained pytorch models",
                   default=["None", "None"])
    p.add_argument("--zsigs", "-zs", nargs="+", default=["zs_hat"])
    p.add_argument("--nb_rir", type=int, default=1, help="number of consecutive RIRs from --rir on")
    p.add_argument("--batch", type=int, default=8, help="RIRs per device call")
    p.add_argument("--dataset", type=str, default=PATH_TO_DATASET, help="root of the data set (holds disco/)")
    p.add_argument("--results", type=str, default="results", help="directory the results/ tree is written under")
    p.add_argument("--online", action="store_true", help="online (recursive) Tango instead of the offline one")
    p.add_argument("--block", type=int, default=8, help="online: frames per filter update")
    p.add_argument("--lag", type=int, default=1, help="online: blocks between statistics and the filter applied")
    return p


def parse_args(argv=None):
    """Command line -> (positional arguments, keyword arguments) of main, converted as tango.py:680-689 does."""
    a = _parser().parse_args(argv)
    models = [None if m == "None" else m for m in a.mods]
    zsigs = a.zsigs[0] if len(a.zsigs) == 1 else a.zsigs
    mask_z = None if a.mask_z == "None" else a.mask_z
    return ((a.vad_type, a.sav_dir, a.rir, a.noise),
            dict(mask_z=mask_z, z_sigs=zsigs, scenario=a.scenario, models=models, nb_rir=a.nb_rir, batch=a.batch,
                 path_to_dataset=a.dataset, results_root=a.results, online=a.online, block=a.block, lag=a.lag))


if __name__ == "__main__":
    args, kwargs = parse_args()
    main(*args, **kwargs)
