// Small elementwise / layout kernels around the hot path.
#include "common.cuh"
#include "kernels.h"

namespace disco {

DISCO_DEV float ipow(float x, int p) {
    float r = 1.f;
    for (int i = 0; i < p; ++i) r *= x;
    return r;
}

// Oracle time-frequency masks, float32 arithmetic like the reference
// (dnn/utils.py:44-71; twin sigproc_utils.py:58-86):
//   kind 0 'irmX': xi = (|s| / max(|n|, eps))^X,  m = xi / (1 + xi)
//   kind 1 'ibmX': m = xi >= 10^(thr/10)                (written as 0.0 / 1.0)
//   kind 2 'iamX': m = (|s| / |s + n|)^X
__global__ void tf_mask_kernel(const float2* __restrict__ S, const float2* __restrict__ Nn, float* __restrict__ M,
                               size_t n, int kind, int power, float thr_lin) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float2 s = S[i], nn = Nn[i];
    const float as = hypotf(s.x, s.y);
    float m;
    if (kind == 2) {
        const float den = hypotf(s.x + nn.x, s.y + nn.y);
        m = ipow(as / den, power);
    } else {
        const float an = fmaxf(hypotf(nn.x, nn.y), 2.220446049250313e-16f);
        const float xi = ipow(as / an, power);
        m = (kind == 0) ? xi / (1.f + xi) : (xi >= thr_lin ? 1.f : 0.f);
    }
    M[i] = m;
}

cudaError_t launch_tf_mask(const float2* S, const float2* Nn, float* M, size_t n, int kind, int power,
                           float thr_lin, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    tf_mask_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(S, Nn, M, n, kind, power, thr_lin);
    return cudaGetLastError();
}

// 32 x 32 tiles: column tiles in grid.x, planes in grid.z; grid.y strides over the row tiles, so a plane of any
// number of rows (T frames of a long recording) fits the 65535 limit of grid.y
template <typename T>
__global__ void transpose_kernel(const T* __restrict__ in, T* __restrict__ out, int rows, int cols) {
    __shared__ T tile[32][33];
    const size_t base = (size_t)blockIdx.z * rows * cols;
    const int c0 = blockIdx.x * 32, row_tiles = (rows + 31) / 32;
    for (int rt = blockIdx.y; rt < row_tiles; rt += gridDim.y) {
        const int r0 = rt * 32;
        for (int i = threadIdx.y; i < 32; i += blockDim.y) {
            const int r = r0 + i, c = c0 + threadIdx.x;
            if (r < rows && c < cols) tile[i][threadIdx.x] = in[base + (size_t)r * cols + c];
        }
        __syncthreads();
        for (int i = threadIdx.y; i < 32; i += blockDim.y) {
            const int c = c0 + i, r = r0 + threadIdx.x;
            if (r < rows && c < cols) out[base + (size_t)c * rows + r] = tile[threadIdx.x][i];
        }
        __syncthreads();   // the tile is refilled by the next row tile
    }
}

template <typename T>
static cudaError_t launch_transpose(const T* in, T* out, int batch, int rows, int cols, cudaStream_t st) {
    if (batch <= 0 || rows <= 0 || cols <= 0) return cudaSuccess;
    const int row_tiles = (rows + 31) / 32;
    dim3 grid((cols + 31) / 32, row_tiles < kMaxGridYZ ? row_tiles : kMaxGridYZ, batch), block(32, 8);
    transpose_kernel<T><<<grid, block, 0, st>>>(in, out, rows, cols);
    return cudaGetLastError();
}
cudaError_t launch_transpose_c64(const float2* in, float2* out, int batch, int rows, int cols, cudaStream_t st) {
    return launch_transpose<float2>(in, out, batch, rows, cols, st);
}
cudaError_t launch_transpose_f32(const float* in, float* out, int batch, int rows, int cols, cudaStream_t st) {
    return launch_transpose<float>(in, out, batch, rows, cols, st);
}

// out = m * in (or (1 - m) * in); the mask plane of a group is shared by its `chans` channels:
// in / out [n_grp][chans][plane], m [n_grp][plane]
__global__ void apply_mask_kernel(const float2* __restrict__ in, const float* __restrict__ m,
                                  float2* __restrict__ out, size_t n, size_t plane, int chans, int one_minus) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const size_t mi = chans == 1 ? i : (i / (plane * chans)) * plane + i % plane;
    float w = m[mi];
    if (one_minus) w = 1.f - w;
    out[i] = cscale(in[i], w);
}
cudaError_t launch_apply_mask(const float2* in, const float* m, float2* out, size_t n, size_t plane, int chans,
                              int one_minus, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    apply_mask_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(in, m, out, n, plane, chans, one_minus);
    return cudaGetLastError();
}

}  // namespace disco
