/* disco_b200 -- C ABI of the H100-native multichannel-Wiener-filter beamforming path.
 *
 * Drop-in boundary for the hot path of nfurnon/disco (reference paths relative to the
 * reference repository root).  The reference has no FFI of its own: its boundary is a set of
 * in-process Python functions.  Each entry point below names the reference interface it
 * replaces; the Python-side binding (ctypes) that mirrors those signatures is
 * disco_b200/_lib.py + disco_b200/ops.py, and INTEGRATION.md shows the stub a maintainer of
 * the reference would add.
 *
 * Conventions
 *   - All array arguments are DEVICE pointers unless the function name ends in _host.
 *   - complex64 = interleaved (re, im) float32 pairs ("float2").
 *   - Spectra are FRAME-MAJOR: [signal][T frames][F = n_fft/2 + 1 bins], bins contiguous.
 *     (The reference's NumPy arrays are (F, T) with T contiguous; layout flags select that
 *     layout for masks and final outputs, see DISCO_LAYOUT_*.)
 *   - hop is fixed to n_fft / 2 (reference N_FFT = 512, N_HOP = 256, tango.py:28-29);
 *     n_fft in {256, 512, 1024}.
 *   - `stream` is a cudaStream_t passed as void* (NULL = default stream).  No entry point
 *     synchronises the device; work is ordered on `stream`.
 *   - Return value: 0 on success; DISCO_ERR_* (< 0) for invalid arguments; a positive
 *     cudaError_t value if a CUDA call failed.  disco_last_error() returns a message for the
 *     calling thread.
 *   - There is no CPU fallback: without a CUDA device every compute entry point fails.
 */
#ifndef DISCO_B200_H
#define DISCO_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DISCO_ABI_VERSION 2

#if defined(__GNUC__)
#define DISCO_API __attribute__((visibility("default")))
#else
#define DISCO_API
#endif

#define DISCO_OK 0
#define DISCO_ERR_INVALID (-1)      /* bad size / unsupported parameter                        */
#define DISCO_ERR_UNSUPPORTED (-2)  /* valid in the reference but not implemented here          */
#define DISCO_ERR_WORKSPACE (-3)    /* workspace too small                                      */

/* layouts of (F, T) planes */
#define DISCO_LAYOUT_TF 0 /* frame-major: [T][F], bins contiguous (native)                      */
#define DISCO_LAYOUT_FT 1 /* reference NumPy layout: [F][T], frames contiguous                   */

/* layout of the exchanged compressed signals Z (all nodes of all utterances) */
#define DISCO_Z_UTT_MAJOR 0  /* [n_utt][K][T][F]: what one GPU holding every node produces            */
#define DISCO_Z_NODE_MAJOR 1 /* [K][n_utt][T][F]: what an all-gather over node-owning ranks delivers   */

/* tf_mask kinds (reference dnn/utils.py:44-71 `type` = 'irmX' | 'ibmX' | 'iamX') */
#define DISCO_MASK_IRM 0
#define DISCO_MASK_IBM 1
#define DISCO_MASK_IAM 2

/* intern_filter types (reference se_utils/internal_formulas.py:31-81 `type`) */
#define DISCO_FILTER_GEVD 0
#define DISCO_FILTER_R1_MWF 1
#define DISCO_FILTER_MWF 2

DISCO_API int disco_abi_version(void);
DISCO_API const char* disco_last_error(void);

/* Number of STFT frames for a signal of `length` samples: 1 + length / (n_fft/2)
 * (librosa center=True; equals the reference's 3 + floor((L - N_FFT) / N_HOP), tango.py:287). */
DISCO_API int disco_n_frames(int length, int n_fft);

/* Create the per-device twiddle / window tables for n_fft ahead of time (they are otherwise
 * created on first use, which must not happen inside CUDA-graph capture). */
DISCO_API int disco_init(int n_fft);

/* Leave `n` SMs (0..64, default 0) free of the persistent fused STFT+SCM kernel, which otherwise occupies every SM
 * with one 213 KB-shared-memory CTA: a collective running on another stream (the NCCL all-gather of the compressed
 * signals, reference tango.py:379-386, in node-sharded runs) then finds SMs for its own CTAs and really overlaps.
 * Process-wide; the workspace functions and the kernels of one batch must see the same value. */
DISCO_API int disco_set_reserved_sms(int n);

/* ---- STFT --------------------------------------------------------------------------------
 * Replaces lb.core.stft(x, n_fft, hop_length=n_fft/2, center=True) [pad_mode='reflect', periodic
 * Hann] at reference tango.py:335-337, get_z_signals.py:274-276, post_generator.py:121,
 * math_utils.py:134-140 (my_stft), for n_sig signals at once.
 *   x [n_sig][length] float32  ->  Y [n_sig][T][F] complex64 */
DISCO_API int disco_stft(const float* x, void* Y, int n_sig, int length, int n_fft, void* stream);

/* ---- fused STFT + mask-weighted spatial covariance ---------------------------------------------
 * Replaces, per group (= one array node of one utterance, C microphones):
 *   STFT of the C channels                                  tango.py:335
 *   s_hat = m * Y, n_hat = (1 - m) * Y                      tango.py:347-348
 *   R_ss[f] = mean_t s_hat s_hat^H, R_nn[f] likewise        tango.py:357-364 (np.outer convention
 *                                                           R[i][j] = a_i conj(a_j))
 *   x    [n_grp][C][length] float32
 *   mask [n_grp] planes of (F, T) float32 in `mask_layout`
 *   Y    [n_grp][C][T][F] complex64                (output, materialised: step 2 re-reads it)
 *   Rss, Rnn [n_grp][F][C][C] complex64            (outputs)
 * C <= 8 (n_fft 256 / 512) or C <= 4 (n_fft 1024); disco_stft_scm_supported() tells.  Other shapes:
 * disco_stft + disco_masked_scm.
 * workspace: disco_stft_scm_workspace() bytes of device scratch.  Rss = Rnn = NULL skips the small
 * reduction launch that materialises the matrices: the per-segment partial sums stay in `workspace`
 * and disco_mwf_solve_workspace() (C <= 4) or disco_scm_from_workspace() consume them (same summation
 * order, identical result). */
DISCO_API size_t disco_stft_scm_workspace(int n_grp, int C, int length, int n_fft);
DISCO_API int disco_stft_scm_supported(int n_fft, int C, int n_mask);
DISCO_API int disco_stft_scm(const float* x, const float* mask, int mask_layout, void* Y, void* Rss, void* Rnn,
                   int n_grp, int C, int length, int n_fft, void* workspace, size_t workspace_bytes,
                   void* stream);

/* ---- fused STFT + the SCMs under TWO masks (single-node arrays, both masks known up front) --------
 * For K = 1 the step-2 statistics (reference tango.py:431-440) are taken over the same Y as the step-1
 * statistics (tango.py:357-364), only under mask_w instead of mask_z.  One pass accumulates both sets.
 *   mask_a, mask_b [n_grp] planes in `mask_layout`; C <= 4, n_fft in {256, 512}.
 *   Y [n_grp][C][T][F] complex64, or NULL: no spectrum is stored (the statistics are the same bit for bit).
 *   disco_stft_filter_dual() then transforms x again to apply both filters, so Y is never written or read.
 * The four matrix sets stay in `workspace` (disco_stft_scm2_workspace() bytes) as per-segment partial sums:
 * disco_mwf_solve_workspace2() solves both filter sets from them in one launch; disco_scm_from_workspace()
 * materialises the matrices of one set (set 0 = mask_a, 1 = mask_b; n_set = 2 here, 1 after disco_stft_scm). */
DISCO_API size_t disco_stft_scm2_workspace(int n_grp, int C, int length, int n_fft);
DISCO_API int disco_stft_scm2(const float* x, const float* mask_a, const float* mask_b, int mask_layout, void* Y,
                    int n_grp, int C, int length, int n_fft, void* workspace, size_t workspace_bytes, void* stream);

/* ---- STFT and both filter-and-sum steps of a single-node array in one pass over the time signals ------
 * disco_filter_dual(W1, W2, disco_stft(x)) without the spectrum in memory: the STFT of every group is computed
 * again and z = w1^H y, zn = y[ref] - z, yf = w2^H y are applied per (frame, bin), with the same arithmetic as
 * disco_filter_dual on the spectrum disco_stft stores (identical results when each group's channels are
 * transformed together, i.e. disco_stft called per group).  Reads 4 C bytes per sample instead of 8 C per bin.
 *   x [n_grp][C][length] float32; W1, W2 [n_grp][F][C] complex64;
 *   z, zn (may be NULL), yf [n_grp] planes in `out_layout` complex64.
 * C <= 4, n_fft in {256, 512} (disco_stft_scm_supported(n_fft, C, 2)). */
DISCO_API int disco_stft_filter_dual(const float* x, const void* W1, const void* W2, void* z, void* zn, void* yf,
                                     int ref, int out_layout, int n_grp, int C, int length, int n_fft, void* stream);
/* disco_scm_from_workspace: Rss, Rnn [n_grp][F][C][C] complex64 out.  It reads disco_stft_scm_workspace() (n_set = 1)
 * or disco_stft_scm2_workspace() (n_set = 2) bytes of `workspace` for (n_grp, C, length, n_fft), laid out by the launch
 * plan of the reserved-SM setting current at the call: the workspace must have been written with the same arguments
 * under the same setting (the library receives no byte count to check). */
DISCO_API int disco_scm_from_workspace(const void* workspace, int n_set, int set, void* Rss, void* Rnn, int n_grp,
                             int C, int length, int n_fft, void* stream);

/* ---- oracle time-frequency masks ----------------------------------------------------------------
 * Replaces tf_mask(s, n, type, bin_thr) (reference dnn/utils.py:44-71, sigproc_utils.py:58-86).
 * Elementwise over n_elem points; `bin_thr_db` as in the reference (dB); ibm is written 0.0/1.0. */
DISCO_API int disco_tf_mask(const void* S, const void* N, float* M, size_t n_elem, int kind, int power,
                  float bin_thr_db, void* stream);

/* ---- mask-weighted SCM of spectra already in HBM (Tango step 2) ---------------------------------
 * Replaces concatenate_signals + the global SCM loops (reference tango.py:142-155, 431-440) with
 * mask_for_z = 'local': group g = (utterance b, node k) sees D = C + K - 1 channels: its own
 * Y[g][0..C), then Z[b][j] for j != k in node order.  K = 1 (Z may be NULL) is the plain
 * masked_scm of SURVEY.md 8(b).  mask == NULL: unweighted SCM into Rss, Rnn zero-filled.
 * Ragged arrays (reference tango.py:259-260, 284: nodes may have different channel counts):
 * launch once per channel count with node_sel = the ascending HOST array of the n_sel node
 * indices that have C microphones (Y, mask, outputs then hold n_utt * n_sel groups);
 * node_sel == NULL means all K nodes.
 *   Y [n_utt*K][C][T][F], Z [n_utt][K][T][F] complex64; mask [n_utt*K] planes; Rss/Rnn [n_utt*K][F][D][D]
 *   (with node_sel: n_utt*n_sel groups in Y, mask and the outputs; Z keeps all K nodes).  F = n_fft/2 + 1 always:
 *   spectra of another bin count are read past their end.
 * z_layout = DISCO_Z_NODE_MAJOR reads Z as [K][n_utt][T][F] -- the buffer an NCCL all-gather over node-owning
 * ranks fills (the reference's exchange, tango.py:379-386) -- so the gathered signals are never transposed. */
DISCO_API int disco_masked_scm(const void* Y, const void* Z, const float* mask, int mask_layout, void* Rss, void* Rnn,
                     int n_utt, int K, int C, int T, int n_fft, const int* node_sel, int n_sel, int z_layout,
                     void* stream);

/* ---- fused step-1 filter-and-sum + step-2 masked SCM for single-node groups (K = 1) ----------------
 * One pass over Y instead of two: z = w1^H y and zn = y[ref] - z (reference tango.py:369-376) are
 * written while the step-2 SCMs under `mask` (= mask_w, tango.py:431-440 with no exchanged signals,
 * D = C) are accumulated.  W1 [n_grp][F][C]; z_out, zn_out [n_grp][T][F] (zn_out may be NULL);
 * Rss, Rnn [n_grp][F][C][C]. */
DISCO_API int disco_filter_sum_scm(const void* W1, const void* Y, const float* mask, int mask_layout, void* z_out,
                                   void* zn_out, int ref, void* Rss, void* Rnn, int n_grp, int C, int T, int n_fft,
                                   void* stream);

/* ---- fused middle pass for multi-node arrays (K > 1) ---------------------------------------------------
 * One pass over Y per utterance: z_k = w1_k^H y_k and zn_k = y_k[ref] - z_k for every node
 * (reference tango.py:369-376), the exchange (every node sees the z of the others, tango.py:379-386)
 * through shared memory, and the step-2 SCMs of every node under its mask_w (tango.py:431-440,
 * mask_for_z = 'local').  Equivalent to disco_filter_sum + disco_masked_scm, reading Y once.
 *   W1 [n_utt*K][F][C]; Y [n_utt*K][C][T][F]; mask_w [n_utt*K][T][F] (frame-major);
 *   Z, ZN [n_utt][K][T][F] (ZN may be NULL); Rss, Rnn [n_utt*K][F][D][D], D = C + K - 1.
 * Available for the (C, K) combinations disco_tango_mid_supported() reports. */
DISCO_API int disco_tango_mid_supported(int C, int K);
DISCO_API int disco_tango_mid(const void* W1, const void* Y, const float* mask_w, void* Z, void* ZN, int ref,
                              void* Rss, void* Rnn, int n_utt, int K, int C, int T, int n_fft, void* stream);

/* ---- per-bin MWF solve ---------------------------------------------------------------------------
 * Replaces intern_filter(Rxx, Rnn, mu, type, rank) (reference internal_formulas.py:31-81) for
 * n_mat matrices: Rss, Rnn [n_mat][D][D] complex64 -> W [n_mat][D], T1 [n_mat][D] complex64
 * (T1 may be NULL).  rank <= 0 means 'full'.  D <= 16.  Arithmetic in float64. */
DISCO_API int disco_mwf_solve(const void* Rss, const void* Rnn, void* W, void* T1, int n_mat, int D, int filter_type,
                    int rank, double mu, void* stream);

/* Same solve, reading the SCMs from the workspace a preceding disco_stft_scm(n_grp, C, length, n_fft) call
 * left behind (matrix index = group * F + bin; W, T1 [n_grp][F][C]).  Rss / Rnn non-NULL: also write the
 * matrices ([n_grp][F][C][C]).  It reads disco_stft_scm_workspace(n_grp, C, length, n_fft) bytes of `workspace` (two
 * sets: disco_stft_scm2_workspace()) as laid out under the current disco_set_reserved_sms value, which must be the one
 * the workspace was written under. */
DISCO_API int disco_mwf_solve_workspace(const void* workspace, void* W, void* T1, void* Rss, void* Rnn, int n_grp,
                                        int C, int length, int n_fft, int filter_type, int rank, double mu,
                                        void* stream);
/* Both filter sets of a disco_stft_scm2() workspace in one launch: W, T1 [2][n_grp][F][C]
 * (set 0 = step-1 filters from mask_a's statistics, set 1 = step-2 filters from mask_b's). */
DISCO_API int disco_mwf_solve_workspace2(const void* workspace, void* W, void* T1, int n_grp, int C, int length,
                               int n_fft, int filter_type, int rank, double mu, void* stream);


/* ---- filter-and-sum ------------------------------------------------------------------------------
 * Replaces np.inner(conj(w), x[:, f, t]) (conj_w = 1) / np.inner(t1, x[:, f, t]) (conj_w = 0) over
 * all (f, t) (reference tango.py:369-374, 445-450) on the same concatenated channel view as
 * disco_masked_scm, and optionally resid = x[ref] - out (zn, tango.py:376).
 *   W [n_utt*K][F][D]; Y, Z as disco_masked_scm; out, resid [n_utt*K] planes in `out_layout` (resid may be NULL);
 *   n_utt*n_sel groups with node_sel */
DISCO_API int disco_filter_sum(const void* W, int conj_w, const void* Y, const void* Z, void* out, void* resid, int ref,
                     int out_layout, int n_utt, int K, int C, int T, int n_fft, const int* node_sel, int n_sel,
                     int z_layout, void* stream);

/* ---- both filter-and-sum steps of a single-node array in one pass over Y ---------------------------
 * Replaces np.inner(conj(w_loc), y) + zn = y[ref] - z (reference tango.py:369-376) AND
 * np.inner(conj(w_glo), y) (tango.py:445-450 with K = 1: no exchanged signals) for every (f, t):
 *   W1, W2 [n_grp][F][C]; Y [n_grp][C][T][F]  ->  z, zn (may be NULL), yf [n_grp] planes in `out_layout`.
 * C <= 4. */
DISCO_API int disco_filter_dual(const void* W1, const void* W2, const void* Y, void* z, void* zn, void* yf, int ref,
                      int out_layout, int n_grp, int C, int T, int n_fft, void* stream);

/* ---- inverse STFT --------------------------------------------------------------------------------
 * Replaces lb.core.istft(S, hop_length=n_fft/2, win_length=n_fft, center=True, length=length)
 * (reference tango.py:528-539, math_utils.py:143-152 my_istft).
 *   Y [n_sig][T][F] complex64 (frame-major) -> x [n_sig][length] float32 */
DISCO_API int disco_istft(const void* Y, float* x, int n_sig, int T, int length, int n_fft, void* stream);

/* ---- STFT / iSTFT of signals of different lengths ---------------------------------------------------
 * A batch of n_sig signals held in rows of `length` samples, signal s being lengths[s] samples long and zero after
 * that (n_fft/2 < lengths[s] <= length).  It has T_s = 1 + lengths[s] / hop frames.
 * disco_stft_lengths: x [n_sig][length] -> Y [n_sig][T][F], T = 1 + length / hop.  Frame t < T_s is disco_stft's
 *   frame of the signal trimmed to lengths[s] (reflect padding at ITS end); frames T_s .. T - 1 are 0.  Signals 2p and
 *   2p + 1 share one complex transform as in disco_stft, so a frame is bit-identical to disco_stft of the trimmed
 *   pair when both signals of the pair have the same length.
 * disco_istft_lengths: Y [n_sig][T][F] -> x [n_sig][length].  Samples < lengths[s] are disco_istft of frames
 *   [0, min(T, T_s)) of signal s to lengths[s] samples (bit-identical when both signals of the pair have the same
 *   length; a pair of different lengths runs each signal alone, as disco_istft runs a single signal); samples from
 *   lengths[s] on are 0.
 * `lengths` is the device copy of the lengths the kernels read; `lengths_host` holds the same values in host memory
 * and is checked before anything is launched (DISCO_ERR_INVALID for a length out of range or a NULL pointer). */
DISCO_API int disco_stft_lengths(const float* x, const int* lengths, const int* lengths_host, void* Y, int n_sig,
                                 int length, int n_fft, void* stream);
DISCO_API int disco_istft_lengths(const void* Y, const int* lengths, const int* lengths_host, float* x, int n_sig,
                                  int T, int length, int n_fft, void* stream);

/* ---- recursive (online) statistics and block-wise filtering ------------------------------------------
 * disco_scm_recursive evaluates, for every frame t and bin, the reference's one-frame update
 *   spatial_correlation_matrix(Rxx, x, lambda_cor, M):  R <- lambda R + (1 - lambda) [M] x x^H
 * (se_utils/internal_formulas.py:84-103) for the pair (R_ss, R_nn) on the concatenated channel view of
 * disco_masked_scm, as a two-level scan, and returns the matrices after the last frame of every block of
 * `block` frames (1..64):  Rss, Rnn [n_utt*n_sel][J][F][D][D], J = ceil(T / block), D = C + K - 1 <= 16.
 * Every entry is the same float32 value at every D, batch position and launch geometry: A_j = the sequential sum
 * over block j's frames in frame order, R_j = fmaf(lambda^(frames of block j), R_(j-1), A_j).  A call on frames
 * [jP, T) with R0 = the matrices after block j - 1 returns the whole call's blocks j, j + 1, ... bit for bit.
 *   weight_power 2: weights m^2 and (1-m)^2 (the caller would pass x = m y, (1-m) y with M = None);
 *   weight_power 1: weights m and 1-m       (x = mixture, M = mask);   mask NULL: weight 1 into Rss, Rnn decays.
 *   R0ss, R0nn: optional initial matrices [n_utt*n_sel][F][D][D] (NULL = zeros), Hermitian.  At D <= 8 every entry
 *   is read; at D >= 9 only the upper triangle (r <= c) and of the diagonal only the real part, the rest is taken
 *   as the conjugate mirror and 0.  (Both agree on an exactly Hermitian R0 with a real diagonal.)
 * disco_filter_sum_blocks applies one filter per block, W [n_utt*n_sel][J][F][D]; out, resid [n_utt*n_sel][T][F]
 * (Y, Z as disco_masked_scm): frame t gets W[.., t / block - lag, ..]
 * (lag = 1: the filter of the last completed block, strictly causal; while that index is negative the
 * reference channel passes through), out = w^H x (conj_w = 1), resid = x[ref] - out (optional). */
DISCO_API int disco_scm_recursive(const void* Y, const void* Z, const float* mask, const void* R0ss, const void* R0nn,
                     void* Rss, void* Rnn, double lambda_cor, int block, int weight_power, int n_utt, int K, int C,
                     int T, int n_fft, const int* node_sel, int n_sel, void* stream);
DISCO_API int disco_filter_sum_blocks(const void* W, int conj_w, const void* Y, const void* Z, void* out, void* resid,
                     int ref, int block, int lag, int n_utt, int K, int C, int T, int n_fft, const int* node_sel,
                     int n_sel, void* stream);
/* The same two calls on utterances of their own lengths: utterance b (every node of it) has frames[b] frames,
 * 1 <= frames[b] <= T, and J_b = ceil(frames[b] / block) blocks; Y, Z and the mask keep their T-frame rows.
 * disco_scm_recursive_lengths: blocks j < J_b are disco_scm_recursive of that utterance alone (its frames [0,
 *   frames[b]) as a call with T = frames[b]) bit for bit -- the last block ends at frames[b] and decays by
 *   lambda^(its frames) -- and blocks J_b .. J - 1 are exact zeros.  No frame >= frames[b] of Y, Z or the mask is
 *   read.  R0 of the utterance (if given) is used as is, as block -1 of its scan.
 * disco_filter_sum_blocks_lengths: frames t < frames[b] are disco_filter_sum_blocks of that utterance alone and read
 *   only the filters of blocks < J_b; frames t >= frames[b] of out and resid are exact zeros, and neither Y / Z nor
 *   W is read for them.
 * `frames` is the device copy the kernels read; `frames_host` the same values in host memory, checked before
 * anything is launched (DISCO_ERR_INVALID for a count out of range or a NULL pointer). */
DISCO_API int disco_scm_recursive_lengths(const void* Y, const void* Z, const float* mask, const void* R0ss,
                     const void* R0nn, void* Rss, void* Rnn, double lambda_cor, int block, int weight_power, int n_utt,
                     int K, int C, int T, int n_fft, const int* node_sel, int n_sel, const int* frames,
                     const int* frames_host, void* stream);
DISCO_API int disco_filter_sum_blocks_lengths(const void* W, int conj_w, const void* Y, const void* Z, void* out,
                     void* resid, int ref, int block, int lag, int n_utt, int K, int C, int T, int n_fft,
                     const int* node_sel, int n_sel, const int* frames, const int* frames_host, void* stream);

/* ---- streaming STFT / iSTFT (the online Tango session, disco_b200/stream.py) -------------------------
 * disco_stft and disco_istft of signals that arrive chunk by chunk, equal to the whole-signal calls value for value
 * (the same pairing of signals 2p, 2p + 1 into one complex transform, the same operations in the same order).
 * disco_stream_stft computes frames [t0, t0 + n_fr) of n_sig signals whose first `length` samples have arrived:
 *   hist     [n_sig][n_fft] float32: samples [L0 - n_fft, L0) of every signal, L0 = length - n_new (entries before
 *            sample 0 are not read)
 *   chunk    [n_sig][n_new] float32: samples [L0, length) (may be NULL when n_new = 0)
 *   hist_out [n_sig][n_fft] float32: receives samples [length - n_fft, length), the next call's `hist` (NULL: no
 *            update; must not alias hist)
 *   Y        [n_sig][n_fr][F] complex64 out; Y_blk (may be NULL) [n_sig][blk_frames][F] receives the same frames at
 *            slots blk_slot .. blk_slot + n_fr - 1
 * Frame t reads samples [t hop - hop, t hop + hop), reflected at the start (librosa center=True); every sample it
 * reads must have arrived, and frame t0 must start within the history.  final_call = 1 ends the stream at `length`
 * (n_new = 0): the frames are then reflected at the end too, and frame length / hop is the last one.
 * disco_stream_istft turns frames [t0, t0 + n_fr) of n_sig spectra Y [n_sig][n_fr][F] into the hop blocks that
 * become final with them: samples [(max(t0, 1) - 1) hop, (t0 + n_fr - 1) hop), written to x[s - x_first] of rows
 * x_stride floats apart.  carry [n_sig][n_fft / 2] float32 holds the windowed second half of the previous frame
 * (zeros before frame 0) and is updated in place.  final_call = 1 also writes the rest of the signal up to `length`.
 * Positions (length, t0, x_first) are relative to an origin the caller may choose per call: a multiple of the hop,
 * at or before every sample the call reads, writes or carries, and 0 at the stream's start (while frame 0 or the
 * start reflection is reachable).  Only distances from the origin reach the kernels, so the results do not depend on
 * it, and a stream may run past 2^31 samples.  Positions must stay below the stream bound:
 * length <= 2^31 - 1 - n_fft - 1024, (t0 + n_fr) hop and x_first likewise; a record past it is DISCO_ERR_INVALID.
 * The same bound caps `length` of disco_stft, disco_stft_scm(2), disco_stft_filter_dual, disco_istft and their
 * _lengths twins. */
DISCO_API int disco_stream_stft(const float* hist, const float* chunk, float* hist_out, void* Y, void* Y_blk,
                                int n_sig, int n_new, int length, int t0, int n_fr, int blk_frames, int blk_slot,
                                int final_call, int n_fft, void* stream);
DISCO_API int disco_stream_istft(const void* Y, float* carry, float* x, int n_sig, int t0, int n_fr, int length,
                                 int final_call, int x_first, int x_stride, int n_fft, void* stream);
/* The same two calls on a pool of n_slot independent streams of n_sig signals each (disco_b200/stream.py,
 * OnlineTangoPool).  Slot s owns signals [s n_sig, (s + 1) n_sig); signals 2p and 2p + 1 of ONE slot share a transform
 * and an odd last signal runs alone, so every slot's outputs are bit-identical to the single-stream call on that slot
 * alone (n_sig signals), whatever the other slots hold.  Each slot has a record of ints; `slots` is the device copy the
 * kernels read and `slots_host` the same values in host memory, checked before anything is launched with the
 * single-stream checks applied per slot (DISCO_ERR_INVALID).
 * disco_stream_stft_slots, record [n_slot][8] = {length, n_new, t0, n_fr, blk_slot, final, hist_sel, hist_write}:
 *   hist  [2][n_slot][n_sig][n_fft] float32: buffer hist_sel of slot s holds its samples [L0 - n_fft, L0), L0 =
 *         length - n_new; with hist_write = 1 its samples [length - n_fft, length) are written to the other buffer
 *   chunk [n_slot][n_sig][n_max] float32: samples [L0, length) at the start of each row (0 <= n_new <= n_max)
 *   Y     [n_slot][n_sig][f_max][F] complex64 out: frames t0 .. t0 + n_fr - 1 (n_fr <= f_max) at rows 0 .. n_fr - 1
 *   Y_blk (may be NULL) [n_slot][n_sig][blk_frames][F]: the same frames at rows blk_slot .. blk_slot + n_fr - 1
 *   A slot with n_fr = 0 and hist_write = 0 is not touched.
 * disco_stream_istft_slots, record [n_slot][5] = {t0, n_fr, length, final, x_first}:
 *   Y     [n_slot][n_sig][f_max][F]: frames t0 .. t0 + n_fr - 1 of slot s at rows 0 .. n_fr - 1
 *   carry [n_slot][n_sig][n_fft / 2], updated in place
 *   x     [n_slot][n_sig][s_max]: sample i of slot s at i - x_first
 *   A slot with n_fr = 0 that is not final is not touched. */
DISCO_API int disco_stream_stft_slots(float* hist, const float* chunk, void* Y, void* Y_blk, const int* slots,
                                      const int* slots_host, int n_slot, int n_sig, int n_max, int f_max,
                                      int blk_frames, int n_fft, void* stream);
DISCO_API int disco_stream_istft_slots(const void* Y, float* carry, float* x, const int* slots, const int* slots_host,
                                       int n_slot, int n_sig, int f_max, int s_max, int n_fft, void* stream);

/* ---- IIR filter bank + band statistics -------------------------------------------------------------
 * Replaces, for every band i of a filter bank, `y = scipy.signal.lfilter(b[i], a[i], x)` followed by the
 * statistics np.var needs, as the reference's frequency-weighted metrics do per third-octave band
 * (metrics.py:96-110 fw_snr, :264-270 fw_sd).  Float64 direct form II transposed.
 *   x     [n_sig] rows of `length` float32 samples, `row_stride` elements apart
 *   sel   NULL: statistics over the outputs that are != 0 (metrics.py:100 `s_f[i][s_f[i] != 0]`);
 *         else same layout as x: over the samples with sel != 0 (metrics.py:102 `[vad_tar != 0]`)
 *   ba    [n_band][2][order + 1] float64: numerator, then denominator; order in {2, 4, 8, 16}
 *   stats [n_sig][n_band][3] float64 out: count, sum, sum of squares */
DISCO_API int disco_band_stats(const float* x, const float* sel, const double* ba, double* stats, int n_sig, int length,
                     long long row_stride, int n_band, int order, void* stream);

/* ---- BSS-eval source scores (float64) -----------------------------------------------------------------
 * Replaces the projections of mir_eval.separation.bss_eval_sources (called six times per node by the reference's
 * evaluation, tango.py:552-567) for n_set reference sets at once.  For set s with references r_1 .. r_nsrc and every
 * estimate row e of it, A_S holds the references of S delayed by 0 .. flen-1 samples (zero-padded), P_S e is the
 * least-squares projection of e onto A_S, and ‖P_S e‖² = ‖y_S‖², L_S y_S = A_S^T e, L_S L_S^T = A_S^T A_S.
 *   refs  [n_set][nsrc][length] float32, ests [n_set][n_est][length] float32
 *   norms [n_set][n_est][1 + 2 nsrc] float64 out:
 *         [0]             ‖e‖²
 *         [1 + b]         the part of ‖y_all‖² (all references) from reference b's block, b < nsrc (sum = ‖P_all e‖²)
 *         [1 + nsrc + k]  ‖y_k‖² = ‖P_k e‖² of reference k alone
 * nsrc 1..4 (more: DISCO_ERR_UNSUPPORTED), flen 1..512 (mir_eval uses 512), length >= 1.  A Cholesky pivot below
 * 1e-10 times the largest diagonal entry of the Gram matrix marks its column as linearly dependent: the projection is
 * then onto the span of the remaining columns (what a least-squares solve gives for a singular Gram matrix).
 * workspace: disco_bss_eval_workspace() bytes (0 for invalid sizes); it grows with n_set: batch in chunks. */
DISCO_API size_t disco_bss_eval_workspace(int n_set, int nsrc, int n_est, int length, int flen);
DISCO_API int disco_bss_eval(const float* refs, const float* ests, double* norms, int n_set, int nsrc, int n_est,
                             int length, int flen, void* workspace, size_t workspace_bytes, void* stream);

/* ---- STOI (float64) -------------------------------------------------------------------------------------
 * Classic STOI as pystoi 0.3 computes it (pystoi.stoi.stoi(x, y, fs_sig), called six times per node by the
 * reference's evaluation, tango.py:569-578), for many (clean, degraded) pairs at once.
 *
 * disco_resample_poly: scipy.signal.resample_poly(x, up, down, window=taps) of n_sig rows, float32 in, float64 out.
 *   x [n_sig][length] float32; y [n_sig][ceil(length up / down)] float64 out; taps [n_taps] float64 (scipy's `window`:
 *   the kernel applies the gain `up` itself).  up and down >= 1 must be coprime and not both 1 (scipy returns a copy
 *   then).  Output sample j is sum_n x[n] up taps[(j + r) down - p - n up] with scipy's centring pre-pad
 *   p = down - h % down and r = (h + p) / down, h = (n_taps - 1) / 2.
 *
 * disco_stoi: STOI of 10 kHz float64 signals (resample first at any other rate).
 *   cleans   [n_clean][length] float64, degraded [n_deg][length] float64
 *   pairs    [n_pair][2] int32: (clean index, degraded index); an index out of range gives d = NaN, n_frames = -1
 *   d        [n_pair] float64 out: the score, 1e-5 where fewer than 30 STFT frames remain (pystoi's value; it warns)
 *   n_sel    [n_clean] int32 out: frames (256 samples, every 128) within 40 dB of the clean's loudest frame
 *   n_frames [n_pair] int32 out: STFT frames scored = n_sel of the pair's clean - 1
 * Every clean's selection and band envelopes are computed once however many pairs share it.  length >= 256 (pystoi
 * raises below).  workspace: disco_stoi_workspace() bytes (0 for invalid sizes); it grows with n_clean + n_pair and
 * with length: batch the pairs in chunks. */
DISCO_API int disco_resample_poly(const float* x, double* y, const double* taps, int n_taps, int up, int down,
                                  int n_sig, int length, void* stream);
DISCO_API size_t disco_stoi_workspace(int n_clean, int n_pair, int length);
DISCO_API int disco_stoi(const double* cleans, const double* degraded, const int* pairs, double* d, int* n_sel,
                         int* n_frames, int n_clean, int n_deg, int n_pair, int length, void* workspace,
                         size_t workspace_bytes, void* stream);
/* The same for signals of their own lengths in rows of `length` samples (the rows are zero after them):
 *   disco_resample_poly_lengths: row s is its first lengths[s] samples (1 <= lengths[s] <= length); output samples
 *     < ceil(lengths[s] up / down) are disco_resample_poly's of the trimmed row, the rest of the output row is 0.
 *   disco_stoi_lengths: clean c, and every degraded signal paired with it, is its first lengths[c] samples
 *     (256 <= lengths[c] <= length): the frame selection stops at the last full frame of those, so a pair scores as
 *     disco_stoi on the trimmed signals does.  With lengths[c] = length for every clean it equals disco_stoi.
 * `lengths` is the device copy the kernels read; `lengths_host` the same values in host memory, checked first
 * (DISCO_ERR_INVALID for a length out of range or a NULL pointer). */
DISCO_API int disco_resample_poly_lengths(const float* x, double* y, const double* taps, int n_taps, int up, int down,
                                          int n_sig, int length, const int* lengths, const int* lengths_host,
                                          void* stream);
DISCO_API int disco_stoi_lengths(const double* cleans, const double* degraded, const int* pairs, double* d, int* n_sel,
                                 int* n_frames, int n_clean, int n_deg, int n_pair, int length, const int* lengths,
                                 const int* lengths_host, void* workspace, size_t workspace_bytes, void* stream);

/* ---- layout helpers -------------------------------------------------------------------------------
 * out[b][c][r] = in[b][r][c] for `batch` planes (complex64 / float32).  Used at the Python
 * boundary to move between the reference (F, T) layout and the native (T, F) layout. */
DISCO_API int disco_transpose_c64(const void* in, void* out, int batch, int rows, int cols, void* stream);
DISCO_API int disco_transpose_f32(const float* in, float* out, int batch, int rows, int cols, void* stream);
/* out = m * in (one_minus = 0) or (1 - m) * in (one_minus = 1), elementwise (tango.py:397-398, 402-403) */
DISCO_API int disco_apply_mask(const void* in, const float* m, void* out, size_t n_elem, int one_minus, void* stream);
/* The same with one mask plane per group shared by its `chans` channels (s_hat_w / n_hat_w of every microphone of a
 * node under the node's mask_w, reference tango.py:413-414): in, out [n_grp][chans][plane], m [n_grp][plane]. */
DISCO_API int disco_apply_mask_channels(const void* in, const float* m, void* out, size_t n_grp, int chans, size_t plane,
                              int one_minus, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DISCO_B200_H */
