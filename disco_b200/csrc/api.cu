// C ABI of libdisco_b200.so (declared in include/disco_b200.h): argument checking, per-device
// constant tables, launch-geometry choices.  No torch types cross this boundary.
#include <limits.h>
#include <math.h>
#include <stdlib.h>
#include <stdio.h>
#include <string.h>

#include <map>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/disco_b200.h"
#include "kernels.h"

using namespace disco;

namespace disco {
// SM count of the CURRENT device (cached per device: processes may drive several GPUs)
int sm_count() {
    static int cache[64] = {0};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
    if (cache[dev] == 0) {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
        cache[dev] = n;
    }
    return cache[dev];
}

}  // namespace disco

namespace {

thread_local std::string g_err;

int fail(int code, const char* msg) {
    g_err = msg;
    return code;
}
int cuda_fail(cudaError_t e, const char* where) {
    g_err = std::string(where) + ": " + cudaGetErrorString(e);
    return (int)e;
}
#define CU(expr, where)                                  \
    do {                                                 \
        cudaError_t _e = (expr);                         \
        if (_e != cudaSuccess) return cuda_fail(_e, where); \
    } while (0)

bool valid_nfft(int n) { return n == 256 || n == 512 || n == 1024; }

// The longest whole signal, and the largest sample position of a stream record, that the STFT / iSTFT kernels address
// in int: they form positions up to a frame and a CTA stride (together < 1024 + n_fft samples) past the signal's end
long long max_length(int n_fft) { return (long long)INT_MAX - n_fft - 1024; }
bool too_long(int length, int n_fft) {
    if (length <= max_length(n_fft)) return false;
    fail(DISCO_ERR_INVALID, "length past 2^31 - 1 - n_fft - 1024 samples");
    return true;
}

struct Tables {
    float2* twiddle = nullptr;   // [N/32][32] W_N^(l k1)
    float* win_half = nullptr;   // 0.5 * periodic Hann (forward: two-for-one split needs the 1/2)
    float* win = nullptr;        // periodic Hann
};
std::mutex g_mu;
std::map<std::pair<int, int>, Tables> g_tables;  // (device, n_fft)

// Build (once per device and n_fft) the twiddle and window tables, computed in double on the host.
int get_tables(int n_fft, Tables* out) {
    int dev = 0;
    CU(cudaGetDevice(&dev), "cudaGetDevice");
    std::lock_guard<std::mutex> lk(g_mu);
    auto key = std::make_pair(dev, n_fft);
    auto it = g_tables.find(key);
    if (it != g_tables.end()) {
        *out = it->second;
        return 0;
    }
    const int RA = n_fft / 32;
    std::vector<float2> tw(n_fft);
    std::vector<float> wh(n_fft), w(n_fft);
    const double two_pi = 6.283185307179586476925286766559;
    for (int k1 = 0; k1 < RA; ++k1)
        for (int l = 0; l < 32; ++l) {
            const double ang = -two_pi * (double)(l * k1) / (double)n_fft;
            tw[k1 * 32 + l] = make_float2((float)cos(ang), (float)sin(ang));
        }
    for (int n = 0; n < n_fft; ++n) {
        const double h = 0.5 - 0.5 * cos(two_pi * (double)n / (double)n_fft);
        w[n] = (float)h;
        wh[n] = (float)(0.5 * h);
    }
    Tables t;
    CU(cudaMalloc(&t.twiddle, n_fft * sizeof(float2)), "cudaMalloc tables");
    CU(cudaMalloc(&t.win_half, n_fft * sizeof(float)), "cudaMalloc tables");
    CU(cudaMalloc(&t.win, n_fft * sizeof(float)), "cudaMalloc tables");
    CU(cudaMemcpy(t.twiddle, tw.data(), n_fft * sizeof(float2), cudaMemcpyHostToDevice), "cudaMemcpy tables");
    CU(cudaMemcpy(t.win_half, wh.data(), n_fft * sizeof(float), cudaMemcpyHostToDevice), "cudaMemcpy tables");
    CU(cudaMemcpy(t.win, w.data(), n_fft * sizeof(float), cudaMemcpyHostToDevice), "cudaMemcpy tables");
    g_tables[key] = t;
    *out = t;
    return 0;
}

// Persistent launch geometry of the fused STFT kernel: one CTA per SM (fewer when there are fewer tiles).
struct StftPlan {
    int n_cta, tiles_per_grp, slots_per_grp;
};
// SMs the persistent fused kernel leaves free (disco_set_reserved_sms): room for the CTAs of a concurrent NCCL
// collective, which cannot co-reside with a 213 KB-shared-memory CTA
int g_reserved_sms = 0;

StftPlan plan_stft(int n_grp, int C, int T, int n_fft) {
    StftPlan pl;
    pl.tiles_per_grp = stft_tiles_per_grp(n_fft, C, T);
    const long long total = (long long)n_grp * pl.tiles_per_grp;
    int sms = sm_count() - g_reserved_sms;
    if (sms < 1) sms = 1;
    pl.n_cta = (int)(total < sms ? total : sms);
    pl.slots_per_grp = stft_slots_per_grp(n_grp, pl.tiles_per_grp, pl.n_cta);
    return pl;
}

size_t stft_ws_bytes(int n_grp, int C, int length, int n_fft, int n_mask) {
    if (!valid_nfft(n_fft) || C < 1 || C > 8 || n_grp < 1 || n_mask < 1) return 0;
    const int T = disco_n_frames(length, n_fft);
    const StftPlan pl = plan_stft(n_grp, C, T, n_fft);
    return (size_t)n_grp * pl.slots_per_grp * n_mask * 2 * C * C * (n_fft / 2 + 1) * sizeof(float);
}

int stft_common(const float* x, const float* mask, const float* mask2, int mask_layout, void* Y, void* Rss,
                void* Rnn, int n_sig, int C, int length, int n_fft, void* workspace, size_t workspace_bytes, int n_mask,
                void* stream) {
    if (!valid_nfft(n_fft)) return fail(DISCO_ERR_INVALID, "n_fft must be 256, 512 or 1024");
    if (n_sig <= 0 || length <= n_fft / 2)
        return fail(DISCO_ERR_INVALID, "need n_sig > 0 and length > n_fft/2 (reflect padding)");
    if (too_long(length, n_fft)) return DISCO_ERR_INVALID;
    if (C < 1) return fail(DISCO_ERR_INVALID, "C must be positive");
    if (!stft_scm_supported(n_fft, C, n_mask))
        return fail(DISCO_ERR_UNSUPPORTED,
                    "fused STFT+SCM: 1..8 channels per group (1..4 with two masks or n_fft = 1024)");
    if (!x || (!Y && n_mask != 2)) return fail(DISCO_ERR_INVALID, "null pointer");   // two masks: Y optional
    Tables tb;
    int rc = get_tables(n_fft, &tb);
    if (rc) return rc;
    const int T = disco_n_frames(length, n_fft);
    const int n_grp = (n_sig + C - 1) / C;
    StftArgs a;
    memset(&a, 0, sizeof(a));
    a.x = x;
    a.mask = mask;
    a.mask2 = mask2;
    a.Y = (float2*)Y;
    a.part = (float*)workspace;
    a.twiddle = tb.twiddle;
    a.window = tb.win_half;
    a.n_sig = n_sig;
    a.n_grp = n_grp;
    a.L = length;
    a.T = T;
    a.mask_ft = (mask_layout == DISCO_LAYOUT_FT);
    a.use_tma = (length % 4 == 0) && ((reinterpret_cast<uintptr_t>(x) & 15) == 0);
    const StftPlan pl = plan_stft(n_grp, C, T, n_fft);
    a.slots_per_grp = pl.slots_per_grp;
    cudaStream_t st = (cudaStream_t)stream;
    if (n_mask > 0) {
        if (!mask || (n_mask == 2 && !mask2) || (!Rss) != (!Rnn)) return fail(DISCO_ERR_INVALID, "null pointer");
        const size_t need = stft_ws_bytes(n_grp, C, length, n_fft, n_mask);
        if (!workspace || workspace_bytes < need) return fail(DISCO_ERR_WORKSPACE, "workspace too small");
    }
    CU(launch_stft_scm(a, n_fft, C, pl.n_cta, n_mask, st), "stft_scm launch");
    if (n_mask == 1 && Rss)
        CU(launch_scm_finalize(a.part, (float2*)Rss, (float2*)Rnn, n_grp, pl.slots_per_grp, pl.tiles_per_grp,
                               pl.n_cta, C, n_fft / 2 + 1, T, 1, 0, st),
           "scm_finalize launch");
    return 0;
}

}  // namespace


extern "C" {

int disco_abi_version(void) { return DISCO_ABI_VERSION; }
const char* disco_last_error(void) { return g_err.c_str(); }

int disco_n_frames(int length, int n_fft) { return 1 + length / (n_fft / 2); }

int disco_set_reserved_sms(int n) {
    if (n < 0 || n > 64) return fail(DISCO_ERR_INVALID, "reserved SMs must be in 0..64");
    g_reserved_sms = n;
    return 0;
}

int disco_init(int n_fft) {
    if (!valid_nfft(n_fft)) return fail(DISCO_ERR_INVALID, "n_fft must be 256, 512 or 1024");
    Tables tb;
    return get_tables(n_fft, &tb);
}

int disco_stft(const float* x, void* Y, int n_sig, int length, int n_fft, void* stream) {
    // plain STFT: signals are grouped by 4 only to share a CTA's tile; groups are independent
    const int C = n_sig >= 4 ? 4 : n_sig;
    return stft_common(x, nullptr, nullptr, 0, Y, nullptr, nullptr, n_sig, C, length, n_fft, nullptr, 0, 0, stream);
}

size_t disco_stft_scm_workspace(int n_grp, int C, int length, int n_fft) {
    return stft_ws_bytes(n_grp, C, length, n_fft, 1);
}

int disco_stft_scm_supported(int n_fft, int C, int n_mask) { return stft_scm_supported(n_fft, C, n_mask) ? 1 : 0; }

int disco_stft_scm(const float* x, const float* mask, int mask_layout, void* Y, void* Rss, void* Rnn, int n_grp,
                   int C, int length, int n_fft, void* workspace, size_t workspace_bytes, void* stream) {
    if (n_grp <= 0) return fail(DISCO_ERR_INVALID, "n_grp must be positive");
    return stft_common(x, mask, nullptr, mask_layout, Y, Rss, Rnn, n_grp * C, C, length, n_fft, workspace,
                       workspace_bytes, 1, stream);
}

size_t disco_stft_scm2_workspace(int n_grp, int C, int length, int n_fft) {
    return stft_ws_bytes(n_grp, C, length, n_fft, 2);
}

int disco_stft_scm2(const float* x, const float* mask_a, const float* mask_b, int mask_layout, void* Y, int n_grp,
                    int C, int length, int n_fft, void* workspace, size_t workspace_bytes, void* stream) {
    if (n_grp <= 0) return fail(DISCO_ERR_INVALID, "n_grp must be positive");
    return stft_common(x, mask_a, mask_b, mask_layout, Y, nullptr, nullptr, n_grp * C, C, length, n_fft, workspace,
                       workspace_bytes, 2, stream);
}

int disco_stft_filter_dual(const float* x, const void* W1, const void* W2, void* z, void* zn, void* yf, int ref,
                           int out_layout, int n_grp, int C, int length, int n_fft, void* stream) {
    if (!valid_nfft(n_fft)) return fail(DISCO_ERR_INVALID, "n_fft must be 256, 512 or 1024");
    if (n_grp < 1 || length <= n_fft / 2)
        return fail(DISCO_ERR_INVALID, "need n_grp > 0 and length > n_fft/2 (reflect padding)");
    if (too_long(length, n_fft)) return DISCO_ERR_INVALID;
    if (!stft_scm_supported(n_fft, C, 2))
        return fail(DISCO_ERR_UNSUPPORTED, "fused STFT+filter: 1..4 channels per group, n_fft 256 or 512");
    if (ref < 0 || ref >= C) return fail(DISCO_ERR_INVALID, "ref channel out of range");
    if (out_layout != DISCO_LAYOUT_TF && out_layout != DISCO_LAYOUT_FT) return fail(DISCO_ERR_INVALID, "bad out_layout");
    if (!x || !W1 || !W2 || !z || !yf) return fail(DISCO_ERR_INVALID, "null pointer");
    Tables tb;
    int rc = get_tables(n_fft, &tb);
    if (rc) return rc;
    const int T = disco_n_frames(length, n_fft);
    StftFilterArgs a;
    memset(&a, 0, sizeof(a));
    a.x = x;
    a.twiddle = tb.twiddle;
    a.window = tb.win_half;
    a.n_sig = n_grp * C;
    a.n_grp = n_grp;
    a.L = length;
    a.T = T;
    a.use_tma = (length % 4 == 0) && ((reinterpret_cast<uintptr_t>(x) & 15) == 0);
    a.W1 = (const float2*)W1;
    a.W2 = (const float2*)W2;
    a.z = (float2*)z;
    a.zn = (float2*)zn;
    a.yf = (float2*)yf;
    a.ref = ref;
    a.out_ft = (out_layout == DISCO_LAYOUT_FT);
    const StftPlan pl = plan_stft(n_grp, C, T, n_fft);
    CU(launch_stft_filter_dual(a, n_fft, C, pl.n_cta, (cudaStream_t)stream), "stft_filter_dual launch");
    return 0;
}

int disco_scm_from_workspace(const void* workspace, int n_set, int set, void* Rss, void* Rnn, int n_grp, int C,
                             int length, int n_fft, void* stream) {
    if (!valid_nfft(n_fft) || n_grp < 1 || C < 1 || C > 8 || n_set < 1 || n_set > 2 || set < 0 || set >= n_set ||
        !workspace || !Rss || !Rnn)
        return fail(DISCO_ERR_INVALID, "bad arguments");
    const int T = disco_n_frames(length, n_fft);
    const StftPlan pl = plan_stft(n_grp, C, T, n_fft);
    CU(launch_scm_finalize((const float*)workspace, (float2*)Rss, (float2*)Rnn, n_grp, pl.slots_per_grp,
                           pl.tiles_per_grp, pl.n_cta, C, n_fft / 2 + 1, T, n_set, set, (cudaStream_t)stream),
       "scm_finalize launch");
    return 0;
}

int disco_tf_mask(const void* S, const void* N, float* M, size_t n_elem, int kind, int power, float bin_thr_db,
                  void* stream) {
    if (kind < 0 || kind > 2) return fail(DISCO_ERR_INVALID, "unknown mask kind");
    if (power < 0 || power > 9) return fail(DISCO_ERR_INVALID, "mask power must be a single digit");
    if (!S || !N || !M) return fail(DISCO_ERR_INVALID, "null pointer");
    const float thr = powf(10.f, bin_thr_db / 10.f);  // math_utils.db2lin
    CU(launch_tf_mask((const float2*)S, (const float2*)N, M, n_elem, kind, power, thr, (cudaStream_t)stream),
       "tf_mask launch");
    return 0;
}

static int make_cat(CatArgs* c, const void* Y, const void* Z, int n_utt, int K, int C, int T, int n_fft,
                    const int* node_sel, int n_sel, int z_layout = DISCO_Z_UTT_MAJOR) {
    if (!valid_nfft(n_fft)) return fail(DISCO_ERR_INVALID, "n_fft must be 256, 512 or 1024");
    if (z_layout != DISCO_Z_UTT_MAJOR && z_layout != DISCO_Z_NODE_MAJOR) return fail(DISCO_ERR_INVALID, "bad z_layout");
    if (n_utt <= 0 || K < 1 || C < 1 || T < 1) return fail(DISCO_ERR_INVALID, "bad sizes");
    if (C + K - 1 > 16) return fail(DISCO_ERR_UNSUPPORTED, "C + K - 1 must be <= 16");
    if (!Y || (K > 1 && !Z)) return fail(DISCO_ERR_INVALID, "null pointer");
    c->Y = (const float2*)Y;
    c->Z = (const float2*)Z;
    c->z_sb = (z_layout == DISCO_Z_NODE_MAJOR) ? 1 : K;
    c->z_sk = (z_layout == DISCO_Z_NODE_MAJOR) ? n_utt : 1;
    c->C = C;
    c->K = K;
    c->T = T;
    c->F = n_fft / 2 + 1;
    if (K > 16) return fail(DISCO_ERR_UNSUPPORTED, "at most 16 nodes");
    if (node_sel) {
        if (n_sel < 1 || n_sel > K) return fail(DISCO_ERR_INVALID, "bad node selection");
        for (int i = 0; i < n_sel; ++i) {
            if (node_sel[i] < 0 || node_sel[i] >= K || (i > 0 && node_sel[i] <= node_sel[i - 1]))
                return fail(DISCO_ERR_INVALID, "node selection must be ascending node indices");
            c->sel[i] = node_sel[i];
        }
        c->n_sel = n_sel;
    } else {
        c->n_sel = K;
        for (int i = 0; i < K; ++i) c->sel[i] = i;
    }
    c->n_grp = n_utt * c->n_sel;
    return 0;
}

int disco_masked_scm(const void* Y, const void* Z, const float* mask, int mask_layout, void* Rss, void* Rnn,
                     int n_utt, int K, int C, int T, int n_fft, const int* node_sel, int n_sel, int z_layout,
                     void* stream) {
    ScmArgs a;
    memset(&a, 0, sizeof(a));
    int rc = make_cat(&a.in, Y, Z, n_utt, K, C, T, n_fft, node_sel, n_sel, z_layout);
    if (rc) return rc;
    if (!Rss || !Rnn) return fail(DISCO_ERR_INVALID, "null pointer");
    if (a.in.n_grp > kMaxGridYZ) return fail(DISCO_ERR_UNSUPPORTED, "at most 65535 (utterance, node) groups per call");
    a.mask = mask;
    a.mask_ft = (mask_layout == DISCO_LAYOUT_FT);
    a.Rss = (float2*)Rss;
    a.Rnn = (float2*)Rnn;
    CU(launch_masked_scm(a, (cudaStream_t)stream), "masked_scm launch");
    return 0;
}

int disco_filter_sum_scm(const void* W1, const void* Y, const float* mask, int mask_layout, void* z_out, void* zn_out,
                         int ref, void* Rss, void* Rnn, int n_grp, int C, int T, int n_fft, void* stream) {
    ScmArgs a;
    memset(&a, 0, sizeof(a));
    int rc = make_cat(&a.in, Y, nullptr, n_grp, 1, C, T, n_fft, nullptr, 0);
    if (rc) return rc;
    if (!W1 || !z_out || !Rss || !Rnn || !mask) return fail(DISCO_ERR_INVALID, "null pointer");
    if (ref < 0 || ref >= C) return fail(DISCO_ERR_INVALID, "ref channel out of range");
    a.mask = mask;
    a.mask_ft = (mask_layout == DISCO_LAYOUT_FT);
    a.Rss = (float2*)Rss;
    a.Rnn = (float2*)Rnn;
    a.W1 = (const float2*)W1;
    a.z_out = (float2*)z_out;
    a.zn_out = (float2*)zn_out;
    a.ref = ref;
    CU(launch_masked_scm(a, (cudaStream_t)stream), "filter_sum_scm launch");
    return 0;
}

int disco_tango_mid_supported(int C, int K) { return tango_mid_supported(C, K) ? 1 : 0; }

int disco_tango_mid(const void* W1, const void* Y, const float* mask_w, void* Z, void* ZN, int ref, void* Rss,
                    void* Rnn, int n_utt, int K, int C, int T, int n_fft, void* stream) {
    if (!valid_nfft(n_fft)) return fail(DISCO_ERR_INVALID, "n_fft must be 256, 512 or 1024");
    if (!W1 || !Y || !mask_w || !Z || !Rss || !Rnn || n_utt < 1 || T < 1)
        return fail(DISCO_ERR_INVALID, "bad arguments");
    if (!tango_mid_supported(C, K)) return fail(DISCO_ERR_UNSUPPORTED, "no fused middle pass for this (C, K)");
    if (ref < 0 || ref >= C) return fail(DISCO_ERR_INVALID, "ref channel out of range");
    MidArgs a;
    a.Y = (const float2*)Y;
    a.W1 = (const float2*)W1;
    a.mask = mask_w;
    a.Z = (float2*)Z;
    a.ZN = (float2*)ZN;
    a.Rss = (float2*)Rss;
    a.Rnn = (float2*)Rnn;
    a.B = n_utt;
    a.K = K;
    a.C = C;
    a.T = T;
    a.F = n_fft / 2 + 1;
    a.ref = ref;
    CU(launch_tango_mid(a, (cudaStream_t)stream), "tango_mid launch");
    return 0;
}

static int solve_workspace(const void* workspace, int n_set, void* W, void* T1, void* Rss, void* Rnn, int n_grp, int C,
                           int length, int n_fft, int filter_type, int rank, double mu, void* stream) {
    if (filter_type < 0 || filter_type > 2) return fail(DISCO_ERR_INVALID, "Unknown filter reference");
    if (!valid_nfft(n_fft) || n_grp < 1 || C < 1 || C > 4 || n_set < 1 || n_set > 2 || !workspace || !W ||
        (!Rss) != (!Rnn))
        return fail(DISCO_ERR_INVALID, "bad arguments");
    const int T = disco_n_frames(length, n_fft), F = n_fft / 2 + 1;
    const StftPlan pl = plan_stft(n_grp, C, T, n_fft);
    SolveArgs a;
    memset(&a, 0, sizeof(a));
    a.Rss = (const float2*)Rss;
    a.Rnn = (const float2*)Rnn;
    a.W = (float2*)W;
    a.T1 = (float2*)T1;
    a.n_mat = n_set * n_grp * F;
    a.n_set = n_set;
    a.D = C;
    a.type = filter_type;
    a.rank = rank;
    a.mu = mu;
    a.part = (const float*)workspace;
    a.slots_per_grp = pl.slots_per_grp;
    a.tiles_per_grp = pl.tiles_per_grp;
    a.n_cta = pl.n_cta;
    a.F = F;
    a.inv_T = 1.0f / (float)T;
    CU(launch_mwf_solve(a, (cudaStream_t)stream), "mwf_solve launch");
    return 0;
}

int disco_mwf_solve_workspace(const void* workspace, void* W, void* T1, void* Rss, void* Rnn, int n_grp, int C,
                              int length, int n_fft, int filter_type, int rank, double mu, void* stream) {
    return solve_workspace(workspace, 1, W, T1, Rss, Rnn, n_grp, C, length, n_fft, filter_type, rank, mu, stream);
}

int disco_mwf_solve_workspace2(const void* workspace, void* W, void* T1, int n_grp, int C, int length, int n_fft,
                               int filter_type, int rank, double mu, void* stream) {
    return solve_workspace(workspace, 2, W, T1, nullptr, nullptr, n_grp, C, length, n_fft, filter_type, rank, mu,
                           stream);
}

int disco_mwf_solve(const void* Rss, const void* Rnn, void* W, void* T1, int n_mat, int D, int filter_type,
                    int rank, double mu, void* stream) {
    if (filter_type < 0 || filter_type > 2) return fail(DISCO_ERR_INVALID, "Unknown filter reference");
    if (D < 1 || D > 16) return fail(DISCO_ERR_UNSUPPORTED, "D must be in 1..16");
    if (n_mat < 0 || !Rss || !Rnn || !W) return fail(DISCO_ERR_INVALID, "bad arguments");
    SolveArgs a;
    memset(&a, 0, sizeof(a));
    a.Rss = (const float2*)Rss;
    a.Rnn = (const float2*)Rnn;
    a.W = (float2*)W;
    a.T1 = (float2*)T1;
    a.n_mat = n_mat;
    a.D = D;
    a.type = filter_type;
    a.rank = rank;
    a.mu = mu;
    CU(launch_mwf_solve(a, (cudaStream_t)stream), "mwf_solve launch");
    return 0;
}

int disco_filter_sum(const void* W, int conj_w, const void* Y, const void* Z, void* out, void* resid, int ref,
                     int out_layout, int n_utt, int K, int C, int T, int n_fft, const int* node_sel, int n_sel,
                     int z_layout, void* stream) {
    FilterArgs a;
    memset(&a, 0, sizeof(a));
    int rc = make_cat(&a.in, Y, Z, n_utt, K, C, T, n_fft, node_sel, n_sel, z_layout);
    if (rc) return rc;
    if (!W || !out) return fail(DISCO_ERR_INVALID, "null pointer");
    if (ref < 0 || ref >= C + K - 1) return fail(DISCO_ERR_INVALID, "ref channel out of range");
    if (a.in.n_grp > kMaxGridYZ) return fail(DISCO_ERR_UNSUPPORTED, "at most 65535 (utterance, node) groups per call");
    a.W = (const float2*)W;
    a.conj_w = conj_w;
    a.out = (float2*)out;
    a.resid = (float2*)resid;
    a.ref = ref;
    a.out_ft = (out_layout == DISCO_LAYOUT_FT);
    CU(launch_filter_sum(a, (cudaStream_t)stream), "filter_sum launch");
    return 0;
}

int disco_filter_dual(const void* W1, const void* W2, const void* Y, void* z, void* zn, void* yf, int ref,
                      int out_layout, int n_grp, int C, int T, int n_fft, void* stream) {
    if (!valid_nfft(n_fft)) return fail(DISCO_ERR_INVALID, "n_fft must be 256, 512 or 1024");
    if (!W1 || !W2 || !Y || !z || !yf || n_grp < 1 || T < 1) return fail(DISCO_ERR_INVALID, "bad arguments");
    if (C < 1 || C > 4) return fail(DISCO_ERR_UNSUPPORTED, "filter_dual supports 1..4 channels");
    if (ref < 0 || ref >= C) return fail(DISCO_ERR_INVALID, "ref channel out of range");
    if (n_grp > 65535) return fail(DISCO_ERR_UNSUPPORTED, "at most 65535 groups per call");
    DualFilterArgs a;
    a.Y = (const float2*)Y;
    a.W1 = (const float2*)W1;
    a.W2 = (const float2*)W2;
    a.z = (float2*)z;
    a.zn = (float2*)zn;
    a.yf = (float2*)yf;
    a.n_grp = n_grp;
    a.C = C;
    a.T = T;
    a.F = n_fft / 2 + 1;
    a.ref = ref;
    a.out_ft = (out_layout == DISCO_LAYOUT_FT);
    CU(launch_filter_dual(a, sm_count(), (cudaStream_t)stream), "filter_dual launch");
    return 0;
}

int disco_istft(const void* Y, float* x, int n_sig, int T, int length, int n_fft, void* stream) {
    if (!valid_nfft(n_fft)) return fail(DISCO_ERR_INVALID, "n_fft must be 256, 512 or 1024");
    if (n_sig <= 0 || T < 1 || length < 1 || !Y || !x) return fail(DISCO_ERR_INVALID, "bad arguments");
    if (too_long(length, n_fft)) return DISCO_ERR_INVALID;
    Tables tb;
    int rc = get_tables(n_fft, &tb);
    if (rc) return rc;
    IstftArgs a;
    memset(&a, 0, sizeof(a));
    a.Y = (const float2*)Y;
    a.x = x;
    a.twiddle = tb.twiddle;
    a.window = tb.win;
    a.n_sig = n_sig;
    a.L = length;
    a.y_frames = T;
    a.ld = length;
    a.j_end = T;
    a.tail = 1;
    CU(launch_istft(a, n_fft, (cudaStream_t)stream), "istft launch");
    return 0;
}

// the per-signal lengths of disco_stft_lengths / disco_istft_lengths: lo < lengths[s] <= hi for every signal
static int check_lengths(const int* lengths_host, int n_sig, int lo, int hi) {
    if (!lengths_host) return fail(DISCO_ERR_INVALID, "null pointer");
    for (int s = 0; s < n_sig; ++s)
        if (lengths_host[s] <= lo || lengths_host[s] > hi)
            return fail(DISCO_ERR_INVALID, "a length is out of range (too short, or longer than the rows)");
    return 0;
}

int disco_stft_lengths(const float* x, const int* lengths, const int* lengths_host, void* Y, int n_sig, int length,
                       int n_fft, void* stream) {
    if (!valid_nfft(n_fft)) return fail(DISCO_ERR_INVALID, "n_fft must be 256, 512 or 1024");
    if (n_sig <= 0 || length <= n_fft / 2)
        return fail(DISCO_ERR_INVALID, "need n_sig > 0 and length > n_fft/2 (reflect padding)");
    if (too_long(length, n_fft)) return DISCO_ERR_INVALID;
    int rc = check_lengths(lengths_host, n_sig, n_fft / 2, length);
    if (rc) return rc;
    if (!x || !lengths || !Y) return fail(DISCO_ERR_INVALID, "null pointer");
    Tables tb;
    rc = get_tables(n_fft, &tb);
    if (rc) return rc;
    StftLengthsArgs a;
    memset(&a, 0, sizeof(a));
    a.x = x;
    a.lengths = lengths;
    a.Y = (float2*)Y;
    a.twiddle = tb.twiddle;
    a.window = tb.win_half;
    a.n_sig = n_sig;
    a.L = length;
    a.T = disco_n_frames(length, n_fft);
    CU(launch_stft_lengths(a, n_fft, (cudaStream_t)stream), "stft_lengths launch");
    return 0;
}

int disco_istft_lengths(const void* Y, const int* lengths, const int* lengths_host, float* x, int n_sig, int T,
                        int length, int n_fft, void* stream) {
    if (!valid_nfft(n_fft)) return fail(DISCO_ERR_INVALID, "n_fft must be 256, 512 or 1024");
    if (n_sig <= 0 || T < 1 || length < 1) return fail(DISCO_ERR_INVALID, "bad arguments");
    if (too_long(length, n_fft)) return DISCO_ERR_INVALID;
    int rc = check_lengths(lengths_host, n_sig, 0, length);
    if (rc) return rc;
    if (!Y || !lengths || !x) return fail(DISCO_ERR_INVALID, "null pointer");
    Tables tb;
    rc = get_tables(n_fft, &tb);
    if (rc) return rc;
    IstftArgs a;
    memset(&a, 0, sizeof(a));
    a.Y = (const float2*)Y;
    a.x = x;
    a.twiddle = tb.twiddle;
    a.window = tb.win;
    a.n_sig = n_sig;
    a.L = length;
    a.y_frames = T;
    a.ld = length;
    a.j_end = T;
    a.tail = 1;
    CU(launch_istft_lengths(a, lengths, n_fft, (cudaStream_t)stream), "istft_lengths launch");
    return 0;
}

// disco_scm_recursive and, with frames / frames_host, disco_scm_recursive_lengths
static int scm_recursive_common(const void* Y, const void* Z, const float* mask, const void* R0ss, const void* R0nn,
                                void* Rss, void* Rnn, double lambda_cor, int block, int weight_power, int n_utt, int K,
                                int C, int T, int n_fft, const int* node_sel, int n_sel, const int* frames,
                                const int* frames_host, void* stream) {
    OnlineLengthsArgs a;
    memset(&a, 0, sizeof(a));
    int rc = make_cat(&a.in, Y, Z, n_utt, K, C, T, n_fft, node_sel, n_sel);
    if (rc) return rc;
    if (a.in.n_grp > kMaxGridYZ) return fail(DISCO_ERR_UNSUPPORTED, "at most 65535 (utterance, node) groups per call");
    if (!Rss || !Rnn || (!R0ss) != (!R0nn)) return fail(DISCO_ERR_INVALID, "null pointer");
    if (block < 1 || block > 64) return fail(DISCO_ERR_INVALID, "block must be 1..64 frames");
    if (!(lambda_cor >= 0.0 && lambda_cor < 1.0)) return fail(DISCO_ERR_INVALID, "lambda_cor must be in [0, 1)");
    if (weight_power != 1 && weight_power != 2) return fail(DISCO_ERR_INVALID, "weight_power must be 1 or 2");
    if (frames_host) {
        rc = check_lengths(frames_host, n_utt, 0, T);
        if (rc) return rc;
        if (!frames) return fail(DISCO_ERR_INVALID, "null pointer");
    }
    a.mask = mask;
    a.R0ss = (const float2*)R0ss;
    a.R0nn = (const float2*)R0nn;
    a.Rss = (float2*)Rss;
    a.Rnn = (float2*)Rnn;
    a.P = block;
    a.J = (T + block - 1) / block;
    a.power = weight_power;
    double g = 1.0 - lambda_cor;
    for (int k = 0; k < 64; ++k) {
        a.gw[k] = (float)g;
        g *= lambda_cor;
    }
    a.lam_block = (float)pow(lambda_cor, block);
    a.lam_last = (float)pow(lambda_cor, T - (a.J - 1) * block);
    a.frames = frames_host ? frames : nullptr;
    for (int n = 1; n <= block; ++n) a.lam_n[n - 1] = (float)pow(lambda_cor, n);   // as lam_block / lam_last
    CU(launch_scm_recursive(a, (cudaStream_t)stream), "scm_recursive launch");
    return 0;
}

int disco_scm_recursive(const void* Y, const void* Z, const float* mask, const void* R0ss, const void* R0nn, void* Rss,
                        void* Rnn, double lambda_cor, int block, int weight_power, int n_utt, int K, int C, int T,
                        int n_fft, const int* node_sel, int n_sel, void* stream) {
    return scm_recursive_common(Y, Z, mask, R0ss, R0nn, Rss, Rnn, lambda_cor, block, weight_power, n_utt, K, C, T,
                                n_fft, node_sel, n_sel, nullptr, nullptr, stream);
}

int disco_scm_recursive_lengths(const void* Y, const void* Z, const float* mask, const void* R0ss, const void* R0nn,
                                void* Rss, void* Rnn, double lambda_cor, int block, int weight_power, int n_utt, int K,
                                int C, int T, int n_fft, const int* node_sel, int n_sel, const int* frames,
                                const int* frames_host, void* stream) {
    if (!frames_host) return fail(DISCO_ERR_INVALID, "null pointer");
    return scm_recursive_common(Y, Z, mask, R0ss, R0nn, Rss, Rnn, lambda_cor, block, weight_power, n_utt, K, C, T,
                                n_fft, node_sel, n_sel, frames, frames_host, stream);
}

// disco_filter_sum_blocks and, with frames / frames_host, disco_filter_sum_blocks_lengths
static int filter_sum_blocks_common(const void* W, int conj_w, const void* Y, const void* Z, void* out, void* resid,
                                    int ref, int block, int lag, int n_utt, int K, int C, int T, int n_fft,
                                    const int* node_sel, int n_sel, const int* frames, const int* frames_host,
                                    void* stream) {
    OnlineFilterArgs a;
    memset(&a, 0, sizeof(a));
    int rc = make_cat(&a.in, Y, Z, n_utt, K, C, T, n_fft, node_sel, n_sel);
    if (rc) return rc;
    if (a.in.n_grp > kMaxGridYZ) return fail(DISCO_ERR_UNSUPPORTED, "at most 65535 (utterance, node) groups per call");
    if (!W || !out) return fail(DISCO_ERR_INVALID, "null pointer");
    if (block < 1 || block > 64 || lag < 0) return fail(DISCO_ERR_INVALID, "bad block / lag");
    if (ref < 0 || ref >= C + K - 1) return fail(DISCO_ERR_INVALID, "ref channel out of range");
    if (frames_host) {
        rc = check_lengths(frames_host, n_utt, 0, T);
        if (rc) return rc;
        if (!frames) return fail(DISCO_ERR_INVALID, "null pointer");
    }
    a.W = (const float2*)W;
    a.conj_w = conj_w;
    a.out = (float2*)out;
    a.resid = (float2*)resid;
    a.ref = ref;
    a.P = block;
    a.J = (T + block - 1) / block;
    a.lag = lag;
    a.frames = frames_host ? frames : nullptr;
    CU(launch_filter_sum_blocks(a, (cudaStream_t)stream), "filter_sum_blocks launch");
    return 0;
}

int disco_filter_sum_blocks(const void* W, int conj_w, const void* Y, const void* Z, void* out, void* resid, int ref,
                            int block, int lag, int n_utt, int K, int C, int T, int n_fft, const int* node_sel,
                            int n_sel, void* stream) {
    return filter_sum_blocks_common(W, conj_w, Y, Z, out, resid, ref, block, lag, n_utt, K, C, T, n_fft, node_sel,
                                    n_sel, nullptr, nullptr, stream);
}

int disco_filter_sum_blocks_lengths(const void* W, int conj_w, const void* Y, const void* Z, void* out, void* resid,
                                    int ref, int block, int lag, int n_utt, int K, int C, int T, int n_fft,
                                    const int* node_sel, int n_sel, const int* frames, const int* frames_host,
                                    void* stream) {
    if (!frames_host) return fail(DISCO_ERR_INVALID, "null pointer");
    return filter_sum_blocks_common(W, conj_w, Y, Z, out, resid, ref, block, lag, n_utt, K, C, T, n_fft, node_sel,
                                    n_sel, frames, frames_host, stream);
}

// Stream records hold positions relative to an origin of the caller's choice (a multiple of the hop, 0 at the stream's
// start), so only their distances matter; every position a kernel forms from an accepted record stays below
// max_length(n_fft).  The checks run in 64 bits, so no field of a record can wrap them.
//
// A stream STFT record against the buffers it addresses: chunk rows of n_max samples, f_max frame rows of Y, and
// (Y_blk) blk_frames rows of the block buffer
static int check_stft_record(const StftSlot& r, int n_fft, int n_max, int f_max, int blk_frames, const void* chunk,
                             const void* Y, const void* Y_blk) {
    typedef long long i64;
    if (r.n_new < 0 || r.n_new > n_max || r.length < r.n_new || r.t0 < 0 || r.n_fr < 0 || r.n_fr > f_max ||
        (r.hist_sel != 0 && r.hist_sel != 1))
        return fail(DISCO_ERR_INVALID, "bad sizes");
    const i64 H = n_fft / 2;
    if (r.length > max_length(n_fft) || ((i64)r.t0 + r.n_fr) * H > max_length(n_fft))
        return fail(DISCO_ERR_INVALID, "positions past 2^31 - 1 - n_fft - 1024 samples: rebase the record");
    if ((r.n_new > 0 && !chunk) || (r.n_fr > 0 && !Y) || (r.final_call && r.n_new > 0))
        return fail(DISCO_ERR_INVALID, "null pointer (or a chunk on the final call)");
    if (r.n_fr > 0) {
        // every sample the frames read has arrived (the last frame is reflected at the end on the final call), and
        // the first one lies within the carried history
        const i64 L0 = (i64)r.length - r.n_new, t1 = (i64)r.t0 + r.n_fr - 1;
        const bool arrived = r.length > H && (r.final_call ? t1 <= r.length / H : (t1 == 0 || (t1 + 1) * H <= r.length));
        if (!arrived || (r.t0 >= 1 && (r.t0 - 1) * H < L0 - n_fft))
            return fail(DISCO_ERR_INVALID, "frames not complete, or older than the carried history");
        if (Y_blk && (r.blk_slot < 0 || (i64)r.blk_slot + r.n_fr > blk_frames))
            return fail(DISCO_ERR_INVALID, "frames outside the block buffer");
    }
    return 0;
}

// A stream iSTFT record against the buffers it addresses: f_max frame rows of Y and rows of s_max samples of x
static int check_istft_record(const IstftSlot& r, int n_fft, int f_max, int s_max, const void* Y, const float* x) {
    typedef long long i64;
    if (r.t0 < 0 || r.n_fr < 0 || r.n_fr > f_max || r.x_first < 0 || (r.length < 1 && (r.n_fr > 0 || r.final_call)))
        return fail(DISCO_ERR_INVALID, "bad sizes");
    const i64 H = n_fft / 2;
    if (r.length > max_length(n_fft) || r.x_first > max_length(n_fft) ||
        ((i64)r.t0 + r.n_fr) * H > max_length(n_fft))
        return fail(DISCO_ERR_INVALID, "positions past 2^31 - 1 - n_fft - 1024 samples: rebase the record");
    if (r.n_fr > 0 && !Y) return fail(DISCO_ERR_INVALID, "null pointer");
    if (r.n_fr <= 0 && !r.final_call) return 0;   // not run
    // samples written: the hop blocks max(t0, 1) .. t0 + n_fr - 1, and on the final call the rest up to length
    const i64 lo = (r.t0 > 0 ? r.t0 - 1 : 0) * H;
    i64 hi = r.final_call ? r.length : ((i64)r.t0 + r.n_fr - 1) * H;
    if (hi > r.length) hi = r.length;
    if (hi > lo) {
        if (!x) return fail(DISCO_ERR_INVALID, "null pointer");
        if (lo < r.x_first || hi > (i64)r.x_first + s_max) return fail(DISCO_ERR_INVALID, "output samples outside x");
    }
    return 0;
}

// disco_stream_stft is one slot whose record is passed by value: the history is read from `hist` (hist_sel = 0) and
// written to hist_out when there is one
int disco_stream_stft(const float* hist, const float* chunk, float* hist_out, void* Y, void* Y_blk, int n_sig,
                      int n_new, int length, int t0, int n_fr, int blk_frames, int blk_slot, int final_call, int n_fft,
                      void* stream) {
    if (!valid_nfft(n_fft)) return fail(DISCO_ERR_INVALID, "n_fft must be 256, 512 or 1024");
    if (n_sig <= 0 || (n_sig + 1) / 2 > kMaxGridYZ) return fail(DISCO_ERR_INVALID, "n_sig must be in 1..131070");
    if (!hist) return fail(DISCO_ERR_INVALID, "null pointer");
    const StftSlot r = {length, n_new, t0, n_fr, blk_slot, final_call ? 1 : 0, 0, hist_out ? 1 : 0};
    int rc = check_stft_record(r, n_fft, n_new, n_fr, blk_frames, chunk, Y, Y_blk);
    if (rc) return rc;
    Tables tb;
    rc = get_tables(n_fft, &tb);
    if (rc) return rc;
    StreamStftArgs a;
    memset(&a, 0, sizeof(a));
    a.hist[0] = const_cast<float*>(hist);   // hist_sel = 0: read only
    a.hist[1] = hist_out;
    a.chunk = chunk;
    a.Y = (float2*)Y;
    a.Y_blk = (float2*)Y_blk;
    a.twiddle = tb.twiddle;
    a.window = tb.win_half;
    a.one = r;
    a.n_slot = 1;
    a.n_sig = n_sig;
    a.n_max = n_new;
    a.f_max = n_fr;
    a.blk_frames = blk_frames;
    CU(launch_stream_stft_slots(a, n_fft, (cudaStream_t)stream), "stream_stft launch");
    return 0;
}

int disco_stream_istft(const void* Y, float* carry, float* x, int n_sig, int t0, int n_fr, int length, int final_call,
                       int x_first, int x_stride, int n_fft, void* stream) {
    if (!valid_nfft(n_fft)) return fail(DISCO_ERR_INVALID, "n_fft must be 256, 512 or 1024");
    if (n_sig <= 0 || (n_sig + 1) / 2 > kMaxGridYZ) return fail(DISCO_ERR_INVALID, "n_sig must be in 1..131070");
    if (length < 1 || x_stride < 0) return fail(DISCO_ERR_INVALID, "bad sizes");
    if (!carry) return fail(DISCO_ERR_INVALID, "null pointer");
    const IstftSlot r = {t0, n_fr, length, final_call ? 1 : 0, x_first};
    int rc = check_istft_record(r, n_fft, n_fr, x_stride, Y, x);
    if (rc) return rc;
    Tables tb;
    rc = get_tables(n_fft, &tb);
    if (rc) return rc;
    IstftArgs a;
    memset(&a, 0, sizeof(a));
    a.Y = (const float2*)Y;
    a.x = x;
    a.carry = carry;
    a.twiddle = tb.twiddle;
    a.window = tb.win;
    a.n_sig = n_sig;
    a.y_frames = n_fr;
    a.ld = x_stride;
    CU(launch_stream_istft_slots(a, nullptr, r, 1, n_fft, (cudaStream_t)stream), "stream_istft launch");
    return 0;
}

// disco_stream_stft_slots: disco_stream_stft's record check per slot, on the host copy of the records
int disco_stream_stft_slots(float* hist, const float* chunk, void* Y, void* Y_blk, const int* slots,
                            const int* slots_host, int n_slot, int n_sig, int n_max, int f_max, int blk_frames,
                            int n_fft, void* stream) {
    if (!valid_nfft(n_fft)) return fail(DISCO_ERR_INVALID, "n_fft must be 256, 512 or 1024");
    if (n_slot <= 0 || n_slot > kMaxGridYZ) return fail(DISCO_ERR_INVALID, "n_slot must be in 1..65535");
    if (n_sig <= 0 || (n_sig + 1) / 2 > kMaxGridYZ) return fail(DISCO_ERR_INVALID, "n_sig must be in 1..131070");
    if (n_max < 0 || f_max < 0 || blk_frames < 0) return fail(DISCO_ERR_INVALID, "bad sizes");
    if (!slots_host || !slots || !hist) return fail(DISCO_ERR_INVALID, "null pointer");
    const StftSlot* recs = (const StftSlot*)slots_host;
    for (int s = 0; s < n_slot; ++s) {
        const int rc = check_stft_record(recs[s], n_fft, n_max, f_max, blk_frames, chunk, Y, Y_blk);
        if (rc) return rc;
    }
    Tables tb;
    int rc = get_tables(n_fft, &tb);
    if (rc) return rc;
    StreamStftArgs a;
    memset(&a, 0, sizeof(a));
    a.hist[0] = hist;
    a.hist[1] = hist + (size_t)n_slot * n_sig * n_fft;
    a.chunk = chunk;
    a.Y = (float2*)Y;
    a.Y_blk = (float2*)Y_blk;
    a.twiddle = tb.twiddle;
    a.window = tb.win_half;
    a.slots = (const StftSlot*)slots;
    a.n_slot = n_slot;
    a.n_sig = n_sig;
    a.n_max = n_max;
    a.f_max = f_max;
    a.blk_frames = blk_frames;
    CU(launch_stream_stft_slots(a, n_fft, (cudaStream_t)stream), "stream_stft_slots launch");
    return 0;
}

// disco_stream_istft_slots: disco_stream_istft's record check per slot, on the host copy of the records
int disco_stream_istft_slots(const void* Y, float* carry, float* x, const int* slots, const int* slots_host,
                             int n_slot, int n_sig, int f_max, int s_max, int n_fft, void* stream) {
    if (!valid_nfft(n_fft)) return fail(DISCO_ERR_INVALID, "n_fft must be 256, 512 or 1024");
    if (n_slot <= 0 || n_slot > kMaxGridYZ) return fail(DISCO_ERR_INVALID, "n_slot must be in 1..65535");
    if (n_sig <= 0 || (n_sig + 1) / 2 > kMaxGridYZ) return fail(DISCO_ERR_INVALID, "n_sig must be in 1..131070");
    if (f_max < 0 || s_max < 0) return fail(DISCO_ERR_INVALID, "bad sizes");
    if (!slots_host || !slots || !carry) return fail(DISCO_ERR_INVALID, "null pointer");
    const IstftSlot* recs = (const IstftSlot*)slots_host;
    for (int s = 0; s < n_slot; ++s) {
        const int rc = check_istft_record(recs[s], n_fft, f_max, s_max, Y, x);
        if (rc) return rc;
    }
    Tables tb;
    int rc = get_tables(n_fft, &tb);
    if (rc) return rc;
    IstftArgs a;
    memset(&a, 0, sizeof(a));
    a.Y = (const float2*)Y;
    a.x = x;
    a.carry = carry;
    a.twiddle = tb.twiddle;
    a.window = tb.win;
    a.n_sig = n_sig;
    a.y_frames = f_max;
    a.ld = s_max;
    const IstftSlot none = {};
    CU(launch_stream_istft_slots(a, (const IstftSlot*)slots, none, n_slot, n_fft, (cudaStream_t)stream),
       "stream_istft_slots launch");
    return 0;
}

int disco_band_stats(const float* x, const float* sel, const double* ba, double* stats, int n_sig, int length,
                     long long row_stride, int n_band, int order, void* stream) {
    if (!x || !ba || !stats || n_sig < 1 || length < 1 || n_band < 1 || row_stride < length)
        return fail(DISCO_ERR_INVALID, "bad arguments");
    if (order != 2 && order != 4 && order != 8 && order != 16)
        return fail(DISCO_ERR_UNSUPPORTED, "filter order must be 2, 4, 8 or 16");
    BankArgs a;
    a.x = x;
    a.sel = sel;
    a.ba = ba;
    a.stats = stats;
    a.n_sig = n_sig;
    a.L = length;
    a.n_band = n_band;
    a.ldx = row_stride;
    CU(launch_band_stats(a, order, (cudaStream_t)stream), "band_stats launch");
    return 0;
}

static int bss_check(int n_set, int nsrc, int n_est, int length, int flen) {
    if (n_set < 1 || n_est < 1 || length < 1 || nsrc < 1) return fail(DISCO_ERR_INVALID, "bad sizes");
    if (flen < 1 || flen > kBssMaxFlen) return fail(DISCO_ERR_INVALID, "flen must be in 1..512");
    if (nsrc > kBssMaxSrc) return fail(DISCO_ERR_UNSUPPORTED, "bss_eval: at most 4 reference sources");
    if ((long long)n_set * nsrc > 0x7fffffffLL || (nsrc + n_est + 3) / 4 > kMaxGridYZ ||
        (length + kBssSeg - 1) / kBssSeg > kMaxGridYZ)
        return fail(DISCO_ERR_UNSUPPORTED, "bss_eval: too many sets, estimates or samples for one call");
    return 0;
}

size_t disco_bss_eval_workspace(int n_set, int nsrc, int n_est, int length, int flen) {
    if (bss_check(n_set, nsrc, n_est, length, flen)) return 0;
    return bss_ws_doubles(n_set, nsrc, n_est, length, flen) * sizeof(double);
}

int disco_bss_eval(const float* refs, const float* ests, double* norms, int n_set, int nsrc, int n_est, int length,
                   int flen, void* workspace, size_t workspace_bytes, void* stream) {
    int rc = bss_check(n_set, nsrc, n_est, length, flen);
    if (rc) return rc;
    if (!refs || !ests || !norms) return fail(DISCO_ERR_INVALID, "null pointer");
    if (!workspace || workspace_bytes < bss_ws_doubles(n_set, nsrc, n_est, length, flen) * sizeof(double))
        return fail(DISCO_ERR_WORKSPACE, "workspace too small");
    BssArgs a;
    memset(&a, 0, sizeof(a));
    a.refs = refs;
    a.ests = ests;
    a.norms = norms;
    a.part = (double*)workspace;
    a.n_set = n_set;
    a.nsrc = nsrc;
    a.n_est = n_est;
    a.L = length;
    a.flen = flen;
    CU(launch_bss_eval(a, (cudaStream_t)stream), "bss_eval launch");
    return 0;
}

static long long gcd_ll(long long a, long long b) { return b == 0 ? a : gcd_ll(b, a % b); }

static int resample_common(const float* x, double* y, const double* taps, int n_taps, int up, int down, int n_sig,
                           int length, const int* lengths, void* stream) {
    if (n_taps < 1 || up < 1 || down < 1 || n_sig < 1 || length < 1) return fail(DISCO_ERR_INVALID, "bad sizes");
    if (gcd_ll(up, down) != 1 || (up == 1 && down == 1))
        return fail(DISCO_ERR_INVALID, "up and down must be coprime and not both 1");
    const long long n_out = ((long long)length * up + down - 1) / down;
    if (n_out > 0x7fffffffLL || (long long)n_sig * ((n_out + 255) / 256) > 0x7fffffffLL)
        return fail(DISCO_ERR_INVALID, "resample_poly: too many output samples for one call");
    if (!x || !y || !taps) return fail(DISCO_ERR_INVALID, "null pointer");
    ResampleArgs a;
    a.x = x;
    a.y = y;
    a.taps = taps;
    a.lengths = lengths;
    a.n_taps = n_taps;
    a.up = up;
    a.down = down;
    a.n_sig = n_sig;
    a.n_in = length;
    a.n_out = (int)n_out;
    CU(launch_resample_poly(a, (cudaStream_t)stream), "resample_poly launch");
    return 0;
}

int disco_resample_poly(const float* x, double* y, const double* taps, int n_taps, int up, int down, int n_sig,
                        int length, void* stream) {
    return resample_common(x, y, taps, n_taps, up, down, n_sig, length, nullptr, stream);
}

int disco_resample_poly_lengths(const float* x, double* y, const double* taps, int n_taps, int up, int down, int n_sig,
                                int length, const int* lengths, const int* lengths_host, void* stream) {
    if (n_sig < 1 || length < 1) return fail(DISCO_ERR_INVALID, "bad sizes");
    int rc = check_lengths(lengths_host, n_sig, 0, length);
    if (rc) return rc;
    if (!lengths) return fail(DISCO_ERR_INVALID, "null pointer");
    return resample_common(x, y, taps, n_taps, up, down, n_sig, length, lengths, stream);
}

static int stoi_check(int n_clean, int n_deg, int n_pair, int length) {
    if (n_clean < 1 || n_deg < 1 || n_pair < 1) return fail(DISCO_ERR_INVALID, "bad sizes");
    if (length < kStoiFrame) return fail(DISCO_ERR_INVALID, "stoi: signals need at least 256 samples");
    const long long groups = (stoi_n_fr(length) - 1 + 3) / 4;
    if (((long long)n_clean + n_pair) * groups > 0x7fffffffLL)
        return fail(DISCO_ERR_INVALID, "stoi: too many signals or samples for one call");
    return 0;
}

size_t disco_stoi_workspace(int n_clean, int n_pair, int length) {
    if (stoi_check(n_clean, 1, n_pair, length)) return 0;
    return stoi_ws_bytes(n_clean, n_pair, length);
}

static int stoi_common(const double* cleans, const double* degraded, const int* pairs, double* d, int* n_sel,
                       int* n_frames, int n_clean, int n_deg, int n_pair, int length, const int* lengths,
                       void* workspace, size_t workspace_bytes, void* stream) {
    int rc = stoi_check(n_clean, n_deg, n_pair, length);
    if (rc) return rc;
    if (!cleans || !degraded || !pairs || !d || !n_sel || !n_frames) return fail(DISCO_ERR_INVALID, "null pointer");
    if (!workspace || workspace_bytes < stoi_ws_bytes(n_clean, n_pair, length))
        return fail(DISCO_ERR_WORKSPACE, "workspace too small");
    StoiArgs a;
    memset(&a, 0, sizeof(a));
    a.cleans = cleans;
    a.degraded = degraded;
    a.pairs = pairs;
    a.d = d;
    a.n_sel = n_sel;
    a.n_frames = n_frames;
    a.energy = (double*)workspace;
    a.lengths = lengths;
    a.n_clean = n_clean;
    a.n_deg = n_deg;
    a.n_pair = n_pair;
    a.L = length;
    CU(launch_stoi(a, (cudaStream_t)stream), "stoi launch");
    return 0;
}

int disco_stoi(const double* cleans, const double* degraded, const int* pairs, double* d, int* n_sel, int* n_frames,
               int n_clean, int n_deg, int n_pair, int length, void* workspace, size_t workspace_bytes, void* stream) {
    return stoi_common(cleans, degraded, pairs, d, n_sel, n_frames, n_clean, n_deg, n_pair, length, nullptr, workspace,
                       workspace_bytes, stream);
}

int disco_stoi_lengths(const double* cleans, const double* degraded, const int* pairs, double* d, int* n_sel,
                       int* n_frames, int n_clean, int n_deg, int n_pair, int length, const int* lengths,
                       const int* lengths_host, void* workspace, size_t workspace_bytes, void* stream) {
    int rc = stoi_check(n_clean, n_deg, n_pair, length);
    if (rc) return rc;
    rc = check_lengths(lengths_host, n_clean, kStoiFrame - 1, length);
    if (rc) return rc;
    if (!lengths) return fail(DISCO_ERR_INVALID, "null pointer");
    return stoi_common(cleans, degraded, pairs, d, n_sel, n_frames, n_clean, n_deg, n_pair, length, lengths, workspace,
                       workspace_bytes, stream);
}

int disco_transpose_c64(const void* in, void* out, int batch, int rows, int cols, void* stream) {
    if (!in || !out) return fail(DISCO_ERR_INVALID, "null pointer");
    if (batch > kMaxGridYZ) return fail(DISCO_ERR_UNSUPPORTED, "at most 65535 planes per call");
    CU(launch_transpose_c64((const float2*)in, (float2*)out, batch, rows, cols, (cudaStream_t)stream),
       "transpose launch");
    return 0;
}
int disco_transpose_f32(const float* in, float* out, int batch, int rows, int cols, void* stream) {
    if (!in || !out) return fail(DISCO_ERR_INVALID, "null pointer");
    if (batch > kMaxGridYZ) return fail(DISCO_ERR_UNSUPPORTED, "at most 65535 planes per call");
    CU(launch_transpose_f32(in, out, batch, rows, cols, (cudaStream_t)stream), "transpose launch");
    return 0;
}
int disco_apply_mask(const void* in, const float* m, void* out, size_t n_elem, int one_minus, void* stream) {
    if (!in || !m || !out) return fail(DISCO_ERR_INVALID, "null pointer");
    CU(launch_apply_mask((const float2*)in, m, (float2*)out, n_elem, n_elem, 1, one_minus, (cudaStream_t)stream),
       "apply_mask launch");
    return 0;
}
int disco_apply_mask_channels(const void* in, const float* m, void* out, size_t n_grp, int chans, size_t plane,
                              int one_minus, void* stream) {
    if (!in || !m || !out || chans < 1) return fail(DISCO_ERR_INVALID, "bad arguments");
    CU(launch_apply_mask((const float2*)in, m, (float2*)out, n_grp * chans * plane, plane, chans, one_minus,
                         (cudaStream_t)stream),
       "apply_mask launch");
    return 0;
}

}  // extern "C"
