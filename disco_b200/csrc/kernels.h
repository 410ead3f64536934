// Internal launcher interface between the kernel translation units and the C ABI (api.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <type_traits>

namespace disco {

// SM count of the current device (cached per device; api.cu) -- launch heuristics size their grids with it
int sm_count();
// grid.y / grid.z are limited to 65535 blocks
constexpr int kMaxGridYZ = 65535;

struct StftArgs {
    const float* x;         // [n_sig][L] float32 time signals (n_sig = n_grp * C, last group may be short)
    const float* mask;      // SCM only: [n_grp][T][F] (mask_ft = 0) or [n_grp][F][T] (mask_ft = 1)
    const float* mask2;     // two-mask SCM only: the second mask, same layout
    float2* Y;              // [n_sig][T][F] complex64, frame-major
    float* part;            // SCM only: [n_grp][slots_per_grp][n_mask][2 C^2][F] partial sums per (group, CTA) segment
    const float2* twiddle;  // [N/32][32]: W_N^(l*k1)
    const float* window;    // [N]: 0.5 * periodic Hann
    int n_sig, n_grp, L, T;
    int slots_per_grp;
    int mask_ft;
    int use_tma;
};
// The filter pass (launch_stft_filter_dual): z = w1^H y, zn = y[ref] - z, yf = w2^H y of single-node groups.  Its own
// parameter type, so the parameter block (and with it the machine code) of the other instantiations stays as it is.
struct StftFilterArgs : StftArgs {
    const float2* W1;       // [n_grp][F][C]
    const float2* W2;       // [n_grp][F][C]
    float2* z;              // [n_grp][T][F] (out_ft = 0) or [n_grp][F][T] (out_ft = 1)
    float2* zn;             // same layout, or null
    float2* yf;             // same layout
    int ref;
    int out_ft;
};

// n_mask: 0 plain STFT (C <= 4: disco_stft groups its signals by at most 4), 1 STFT + SCMs under `mask`, 2 STFT +
// SCMs under `mask` and `mask2`.  Two masks and Y == null: the statistics only, no spectrum is stored.
cudaError_t launch_stft_scm(const StftArgs& a, int n_fft, int C, int n_cta, int n_mask, cudaStream_t st);
// STFT + both filters of a single-node array per (frame, bin), Y never stored; the coverage of n_mask = 2
cudaError_t launch_stft_filter_dual(const StftFilterArgs& a, int n_fft, int C, int n_cta, cudaStream_t st);
bool stft_scm_supported(int n_fft, int C, int n_mask);
// matrices of mask set `set` (of n_set) from the segment partial sums
cudaError_t launch_scm_finalize(const float* part, float2* Rss, float2* Rnn, int n_grp, int slots_per_grp,
                                int tiles_per_grp, int n_cta, int C, int F, int T, int n_set, int set, cudaStream_t st);
int stft_tile_frames(int n_fft, int C);
int stft_tiles_per_grp(int n_fft, int C, int T);

// Segment layout of the partial sums (StftArgs::part).  The total = n_grp * tiles_per_grp tiles are cut into
// n_cta contiguous ranges, CTA b owning [total * b / n_cta, total * (b + 1) / n_cta); the CTAs whose range meets
// group g write its slots 0, 1, ... in CTA order, and the finalize kernel and the solver sum them in that order.
// first CTA whose tile range contains tile i
__host__ __device__ __forceinline__ int cta_of_tile(long long i, long long total, int n_cta) {
    int b = (int)((i * n_cta) / total);
    if (b >= n_cta) b = n_cta - 1;
    while (b + 1 < n_cta && total * (b + 1) / n_cta <= i) ++b;
    while (b > 0 && total * b / n_cta > i) --b;
    return b;
}
// the CTAs that wrote the slots of group g: first .. last, in slot order
struct SegSlots {
    int first, last;
    __host__ __device__ __forceinline__ int count() const { return last - first + 1; }
};
__host__ __device__ __forceinline__ SegSlots seg_slots(int g, int tiles_per_grp, long long total, int n_cta) {
    return {cta_of_tile((long long)g * tiles_per_grp, total, n_cta),
            cta_of_tile((long long)(g + 1) * tiles_per_grp - 1, total, n_cta)};
}
// Upper bound on the number of CTAs whose tile range intersects one group (slots_per_grp).
inline int stft_slots_per_grp(int n_grp, int tiles_per_grp, int n_cta) {
    const long long total = (long long)n_grp * tiles_per_grp;
    const long long min_range = total / n_cta;   // every CTA owns floor or ceil(total / n_cta) tiles
    if (min_range == 0) return tiles_per_grp + 1;
    return (int)(tiles_per_grp / min_range) + 2;
}

// Step-2 style input: group g = (utterance b, node k) sees D = C + K - 1 channels:
// its own C microphone spectra, then the compressed signals z of the other nodes in node
// order (reference concatenate_signals, tango.py:142-155).
// Ragged arrays (nodes with different microphone counts) are handled by launching once per
// channel count on the subset `sel` of nodes that have C microphones: group g = (b, sel[g % n_sel]).
struct CatArgs {
    const float2* Y;   // [n_grp][C][T][F]
    const float2* Z;   // [n_utt][K][T][F] (z_sb = K, z_sk = 1) or node-major [K][n_utt][T][F] (z_sb = 1, z_sk = n_utt);
                       // may be null when K == 1
    long long z_sb, z_sk;   // plane (T x F) strides of Z along the utterance and the node axis
    int C, K, T, F;
    int n_grp;         // = n_utt * n_sel
    int n_sel;         // nodes covered by this launch (K when all nodes have C microphones)
    int sel[16];       // their node indices, ascending
};

// Plane [T][F] of channel d of group grp: d < C is an own microphone, d >= C the compressed signal of node j, the
// other nodes in order, skipping the group's own node (tango.py:153-155).
__device__ __forceinline__ const float2* cat_channel(const CatArgs& in, int grp, int d) {
    if (d < in.C) return in.Y + ((size_t)grp * in.C + d) * in.T * in.F;
    const int b = grp / in.n_sel, k = in.sel[grp % in.n_sel];
    int j = d - in.C;
    if (j >= k) ++j;
    return in.Z + ((size_t)b * in.z_sb + (size_t)j * in.z_sk) * in.T * in.F;
}

struct ScmArgs {
    CatArgs in;
    const float* mask;   // [n_grp][T][F] or [n_grp][F][T]; null = all ones (plain SCM into Rss, Rnn = 0)
    int mask_ft;
    float2* Rss;         // [n_grp][F][D][D]
    float2* Rnn;
    // optional fused step-1 filter-and-sum (single-node groups, K == 1): z = w1^H y, zn = y[ref] - z
    const float2* W1;    // [n_grp][F][C] or null
    float2* z_out;       // [n_grp][T][F]
    float2* zn_out;      // [n_grp][T][F] or null
    int ref;
};
cudaError_t launch_masked_scm(const ScmArgs& a, cudaStream_t st);
cudaError_t launch_masked_scm_wide(const ScmArgs& a, cudaStream_t st);   // D = 5..16 (scm_wide.cu)

struct SolveArgs {
    const float2* Rss;   // [n_mat][D][D]
    const float2* Rnn;
    float2* W;           // [n_mat][D]
    float2* T1;          // [n_mat][D] (may be null)
    int n_mat, D;
    int type;            // 0 gevd, 1 r1-mwf, 2 mwf
    int rank;            // gevd: number of generalised eigenpairs kept; <= 0 or >= D means full
    double mu;
    // optional, D <= 4 only: read the matrices straight from the fused STFT+SCM kernel's segment partial sums
    // (skips scm_finalize); matrix idx = (set * n_grp + grp) * F + f, n_mat = n_set * n_grp * F
    const float* part;   // [n_grp][slots_per_grp][n_set][2 D^2][F] or null
    int slots_per_grp, tiles_per_grp, n_cta, F;
    int n_set;           // mask sets in the partial sums (0 is read as 1)
    float inv_T;
};
cudaError_t launch_mwf_solve(const SolveArgs& a, cudaStream_t st);

struct FilterArgs {
    CatArgs in;
    const float2* W;     // [n_grp][F][D]
    int conj_w;          // 1: w^H x (reference np.inner(conj(w), x)); 0: w^T x (reference np.inner(t1, x))
    float2* out;         // [n_grp][T][F] (out_ft = 0) or [n_grp][F][T] (out_ft = 1)
    float2* resid;       // optional: in[ref] - out, same layout as out (reference zn, tango.py:376)
    int ref;             // reference channel for resid
    int out_ft;
};
cudaError_t launch_filter_sum(const FilterArgs& a, cudaStream_t st);
cudaError_t launch_filter_sum_multi(const FilterArgs& a, cudaStream_t st);   // K > 1, all nodes, TF output

// Time split of the filter launches (grid.z): frames per slab, a multiple of 32.  When the ctas = bin blocks x
// groups are fewer than want_ctas, the T frames are halved into more slabs while a slab keeps more than 64 frames.
inline int filter_slab_frames(int T, int ctas, int want_ctas) {
    int slabs = 1;
    while (ctas * slabs < want_ctas && (T + slabs - 1) / slabs > 64) slabs *= 2;
    return ((T + slabs - 1) / slabs + 31) / 32 * 32;
}

// Single-node groups, both filters in one pass over Y (filter_dual.cu): z = w1^H y, zn = y[ref] - z, yf = w2^H y
struct DualFilterArgs {
    const float2* Y;     // [n_grp][C][T][F]
    const float2* W1;    // [n_grp][F][C] step-1 filters
    const float2* W2;    // [n_grp][F][C] step-2 filters
    float2* z;           // [n_grp][T][F] (out_ft = 0) or [n_grp][F][T]
    float2* zn;          // same layout, may be null
    float2* yf;          // same layout
    int n_grp, C, T, F, ref, out_ft;
};
cudaError_t launch_filter_dual(const DualFilterArgs& a, int sm_count, cudaStream_t st);

// Fused multi-node middle pass (mid_multi.cu): z, zn of every node + step-2 SCMs of every node.
struct MidArgs {
    const float2* Y;     // [B*K][C][T][F]
    const float2* W1;    // [B*K][F][C]  step-1 filters
    const float* mask;   // [B*K][T][F]  step-2 masks (frame-major only)
    float2* Z;           // [B][K][T][F] out
    float2* ZN;          // [B][K][T][F] out (may be null)
    float2* Rss;         // [B*K][F][D][D] out, D = C + K - 1, reference channel order
    float2* Rnn;
    int B, K, C, T, F, ref;
};
cudaError_t launch_tango_mid(const MidArgs& a, cudaStream_t st);
bool tango_mid_supported(int C, int K);

// Recursive (online) SCMs and block-wise filtering (online.cu; reference internal_formulas.py:84-103).
struct OnlineArgs {
    CatArgs in;
    const float* mask;      // [n_grp][T][F] frame-major, or null (all ones: plain smoothed SCM into Rss, Rnn = decay only)
    const float2* R0ss;     // optional initial matrices [n_grp][F][D][D]
    const float2* R0nn;
    float2* Rss;            // [n_grp][J][F][D][D]: smoothed SCMs after the last frame of every block
    float2* Rnn;
    int P, J;               // frames per block, number of blocks = ceil(T / P)
    int power;              // 2: weights m^2, (1-m)^2 (x = m y estimate, M = None); 1: m, 1-m (x = mixture, M = mask)
    float lam_block, lam_last;   // lambda^P, lambda^(frames of the last block)
    float gw[64];           // (1 - lambda) lambda^k, k = 0..P-1
};
// Utterances of their own lengths: the kernels' template LEN = true take this struct, LEN = false the plain
// OnlineArgs, so the uniform kernels keep their parameter layout.  Utterance b = grp / n_sel has frames[b] <= T
// frames and J_b = ceil(frames[b] / P) blocks; its short last block decays by lam_n[frames - 1]; blocks >= J_b are
// stored as 0.  frames = null runs the uniform kernels.
struct OnlineLengthsArgs : OnlineArgs {
    const int* frames;      // [n_utt] device, or null
    float lam_n[64];        // (float)lambda^n, n = 1..P (lam_n[P - 1] = lam_block)
};
template <bool LEN>
using OnlineParams = std::conditional_t<LEN, OnlineLengthsArgs, OnlineArgs>;
cudaError_t launch_scm_recursive(const OnlineLengthsArgs& a, cudaStream_t st);
// D = 9..16 (online_wide.cu): a CTA per (group, 32-bin block) streams the frames and carries R_(j-1) itself; same
// values as launch_scm_recursive's two-level scan.  Reads of R0: upper triangle, real part of the diagonal.
cudaError_t launch_scm_recursive_wide(const OnlineLengthsArgs& a, cudaStream_t st);

struct OnlineFilterArgs {
    CatArgs in;
    const float2* W;        // [n_grp][J][F][D] one filter per block
    int conj_w;
    float2* out;            // [n_grp][T][F]
    float2* resid;          // optional x[ref] - out
    int ref, P, J, lag;     // frame t uses filter t / P - lag (pass-through of channel `ref` while that is < 0)
    // utterances of their own lengths, or null: utterance b = grp / n_sel has frames[b] <= T frames; frames from
    // frames[b] on are written 0 and the filters of blocks >= ceil(frames[b] / P) are never read
    const int* frames;      // [n_utt] device
};
// a.frames selects the length-aware instantiations (template LEN = true); null runs the uniform kernels
cudaError_t launch_filter_sum_blocks(const OnlineFilterArgs& a, cudaStream_t st);
cudaError_t launch_filter_sum_blocks_wide(const OnlineFilterArgs& a, cudaStream_t st);   // D = 9..16

// IIR filter bank + band statistics (filterbank.cu; reference metrics.py fw_snr / fw_sd).
struct BankArgs {
    const float* x;      // [n_sig] rows of L samples, row stride ldx
    const float* sel;    // optional, same layout: statistics over samples with sel != 0 (else: output != 0)
    const double* ba;    // [n_band][2][order + 1]: numerator b, then denominator a
    double* stats;       // [n_sig][n_band][3]: count, sum, sum of squares of the selected filter outputs
    int n_sig, L, n_band;
    long long ldx;
};
cudaError_t launch_band_stats(const BankArgs& a, int order, cudaStream_t st);

// BSS-eval squared norms (bss.cu; mir_eval.separation.bss_eval_sources as tango.main calls it).
constexpr int kBssMaxSrc = 4;         // references per set
constexpr int kBssMaxFlen = 512;      // mir_eval's filter length
constexpr int kBssSeg = 4096;         // samples per correlation time segment
constexpr double kBssDelta = 1e-10;   // a pivot <= kBssDelta * max diag G marks a dependent column
struct BssArgs {
    const float* refs;   // [n_set][nsrc][L]
    const float* ests;   // [n_set][n_est][L]
    double* norms;       // [n_set][n_est][1 + 2 nsrc]: ‖e‖², ‖y_all‖² per reference block, ‖y_k‖² of each reference alone
    double* part;        // workspace: segment partial correlations, then the rest (set by the launcher)
    double* corr;
    double* mat;
    size_t mat_per_set;
    int n_set, nsrc, n_est, L, flen, n_seg;
};
size_t bss_ws_doubles(int n_set, int nsrc, int n_est, int L, int flen);
cudaError_t launch_bss_eval(BssArgs a, cudaStream_t st);

// Polyphase resampler with scipy.signal.resample_poly's alignment and gain (stoi.cu).
struct ResampleArgs {
    const float* x;      // [n_sig][n_in]
    double* y;           // [n_sig][n_out], n_out = ceil(n_in up / down)
    const double* taps;  // [n_taps] scipy's `window` (the gain `up` is applied in the kernel, as scipy does)
    const int* lengths;  // null, or [n_sig]: signal s is its first lengths[s] <= n_in samples (zero output after
                         // ceil(lengths[s] up / down))
    int n_taps, up, down, n_sig, n_in, n_out;
};
cudaError_t launch_resample_poly(const ResampleArgs& a, cudaStream_t st);

// Classic STOI (pystoi 0.3) of 10 kHz float64 signals (stoi.cu).
constexpr int kStoiFrame = 256;   // frame length; frames start every kStoiFrame / 2 samples
constexpr int kStoiBands = 15;    // one-third octave bands
constexpr int kStoiSeg = 30;      // STFT frames per segment
struct StoiArgs {
    const double* cleans;    // [n_clean][L]
    const double* degraded;  // [n_deg][L]
    const int* pairs;        // [n_pair][2]: clean index, degraded index
    double* d;               // [n_pair]
    int* n_sel;              // [n_clean]: frames kept by the silent-frame removal
    int* n_frames;           // [n_pair]: STFT frames scored (n_sel of the pair's clean - 1; -1 for a bad pair)
    double* energy;          // workspace [n_clean][n_fr]
    int* sel;                // workspace [n_clean][n_fr]: kept frame indices, in order
    double* tob;             // workspace [n_clean + n_pair][n_fr][kStoiBands]: band envelopes
    const int* lengths;      // null, or [n_clean]: clean c (and every degraded signal paired with it) is its first
                             // lengths[c] <= L samples; its frame selection stops at the last full frame of those
    int n_clean, n_deg, n_pair, L, n_fr;
};
int stoi_n_fr(int L);
size_t stoi_ws_bytes(int n_clean, int n_pair, int L);
cudaError_t launch_stoi(StoiArgs a, cudaStream_t st);

// Hop blocks [j_begin, j_end) of the iSTFT of every signal (istft.cu).  Whole signals (launch_istft, carry == null):
// blocks [0, T), the launcher drops those past L and splits the rest into chunks of fpc blocks, each of which
// recomputes the frame before its first block.  A stream (launch_stream_istft_slots, below): the blocks of frames
// t0 .. t0 + n_fr - 1 of its record, one CTA per signal pair, the windowed half frame before them carried in `carry`.
struct IstftArgs {
    const float2* Y;        // frame j of signal s at Y + (s * y_frames + j - y_t0) * F, frame-major complex64
    float* x;               // sample i of signal s at x[s * ld + i - x_first]
    float* carry;           // null, or [n_sig][N/2]: windowed second half of frame j_begin - 1 in, of frame j_end - 1 out
    const float2* twiddle;
    const float* window;    // [N] periodic Hann (unscaled)
    int n_sig, L;           // signals, samples per signal
    int y_frames, y_t0, ld, x_first;
    int j_begin, j_end;
    int fpc;                // blocks per chunk (grid.x); set by the launcher
    int tail;               // 1: also block j_end (second half of frame j_end - 1) and the zero fill up to L
};
cudaError_t launch_istft(const IstftArgs& a, int n_fft, cudaStream_t st);

// Signals of their own lengths in rows of a common length (lengths.cu).  Signal s holds lengths[s] samples
// (hop < lengths[s] <= L) and 1 + lengths[s] / hop frames; the rest of its row (samples, frames) is zero.
struct StftLengthsArgs {
    const float* x;         // [n_sig][L] float32
    const int* lengths;     // [n_sig] device
    float2* Y;              // [n_sig][T][F], T = 1 + L / hop
    const float2* twiddle;  // [N/32][32]
    const float* window;    // [N]: 0.5 * periodic Hann
    int n_sig, L, T;
};
cudaError_t launch_stft_lengths(const StftLengthsArgs& a, int n_fft, cudaStream_t st);
// a: as disco_istft fills it (Y [n_sig][y_frames][F], x [n_sig][L], j_end = y_frames); lengths [n_sig] device
cudaError_t launch_istft_lengths(const IstftArgs& a, const int* lengths, int n_fft, cudaStream_t st);
// istft.cu's per-length kernel (it runs istft_body) and its launch geometry, for launch_istft_lengths
struct IstftLengthsKernel {
    const void* fn;
    int threads;
    size_t smem;
    int items;
};
IstftLengthsKernel istft_lengths_kernel_for(int n_fft);

// Streaming STFT (stream.cu): disco_stft on signals that arrive chunk by chunk, in n_slot independent streams (slots)
// of n_sig signals each.  Slot s owns signals [s n_sig, (s + 1) n_sig) of every buffer and has the record below: from
// the device array `slots` (a pool, disco_stream_stft_slots) or, with slots = null, `one` (n_slot = 1: a lockstep
// stream, disco_stream_stft, whose record travels in the kernel parameters).
struct StftSlot {
    int length, n_new, t0, n_fr, blk_slot;
    int final_call;         // 1: the stream ends at `length` (reflect padding at the end)
    int hist_sel;           // the history buffer read (0 / 1)
    int hist_write;         // 1: samples [length - N, length) are written to the other buffer
};
constexpr int kStftSlotFields = 8;   // ints per record of the C ABI
static_assert(sizeof(StftSlot) == kStftSlotFields * sizeof(int), "StftSlot is the C ABI's record");
struct StreamStftArgs {
    float* hist[2];         // two [n_slot][n_sig][N] buffers: samples [L0 - N, L0) in one, L0 = length - n_new
    const float* chunk;     // [n_slot][n_sig][n_max]: samples [L0, length) at the start of each row
    float2* Y;              // [n_slot][n_sig][f_max][F]: frames t0 .. t0 + n_fr - 1 at rows 0 .. n_fr - 1
    float2* Y_blk;          // optional [n_slot][n_sig][blk_frames][F]: the same frames at rows blk_slot ..
    const float2* twiddle;  // [N/32][32]
    const float* window;    // [N]: 0.5 * periodic Hann
    const StftSlot* slots;  // [n_slot] device, or null: `one`
    StftSlot one;
    int n_slot, n_sig, n_max, f_max, blk_frames;
};
// n_slot slots (a lockstep stream is one); no launch when nothing changes (a by-value record with no frames and no
// history to write)
cudaError_t launch_stream_stft_slots(const StreamStftArgs& a, int n_fft, cudaStream_t st);
// The stream iSTFT (istft.cu): slot s runs istft_body on its signals [s n_sig, (s + 1) n_sig) with its record, from
// `slots` (device, a pool) or, with slots = null, `one` (n_slot = 1, a lockstep stream).  a: Y [n_slot][n_sig]
// [y_frames][F], carry [n_slot][n_sig][N/2], x [n_slot][n_sig][ld]; a.n_sig is the signals of one slot.  A slot with
// n_fr = 0 that is not final is not run.
struct IstftSlot {
    int t0, n_fr, length, final_call, x_first;
};
constexpr int kIstftSlotFields = 5;   // ints per record of the C ABI
static_assert(sizeof(IstftSlot) == kIstftSlotFields * sizeof(int), "IstftSlot is the C ABI's record");
cudaError_t launch_stream_istft_slots(const IstftArgs& a, const IstftSlot* slots, const IstftSlot& one, int n_slot,
                                      int n_fft, cudaStream_t st);

cudaError_t launch_tf_mask(const float2* S, const float2* Nn, float* M, size_t n, int kind, int power,
                           float thr_lin, cudaStream_t st);
// out[b][c][r] = in[b][r][c]
cudaError_t launch_transpose_c64(const float2* in, float2* out, int batch, int rows, int cols, cudaStream_t st);
cudaError_t launch_transpose_f32(const float* in, float* out, int batch, int rows, int cols, cudaStream_t st);
// out = m * in or (1 - m) * in over n = n_grp * chans * plane points; the mask [n_grp][plane] is shared by the
// `chans` channels of a group
cudaError_t launch_apply_mask(const float2* in, const float* m, float2* out, size_t n, size_t plane, int chans,
                              int one_minus, cudaStream_t st);

}  // namespace disco
