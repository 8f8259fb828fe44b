// snn_ops.cu — single-operator entry points of the C ABI (the reference's per-object methods:
// Connection.compute, connection.update, normalize) and the multi-GPU window-combine kernels.
#include "snn_phases.cuh"
#include "snn_combine.cuh"

namespace {

// out[b,j] = sum_{i: s[b,i]} w[i,j] (+ bias).  Connection.compute (topology.py:332-346).
__global__ void __launch_bounds__(SNN_GEN_THREADS) conn_compute_kernel(snn_conn_t C, int ns, int nt, int B,
                                                                        const uint8_t *__restrict__ s, float *__restrict__ out) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int tile = blockIdx.x, j = tile * SNN_TILE + lane;
    const bool valid = j < nt;
    for (int b = blockIdx.y * SNN_GEN_WARPS + warp; b < B; b += gridDim.y * SNN_GEN_WARPS) {
        float p = 0.0f;
        for (int i0 = 0; i0 < ns; i0 += 32) {
            const bool sp = (i0 + lane < ns) && s[(size_t)b * ns + i0 + lane] != 0;
            uint32_t word = __ballot_sync(0xffffffffu, sp);
            while (word) {
                const int i = i0 + __ffs(word) - 1;
                word &= word - 1;
                if (valid) p = p + C.w[(size_t)i * nt + j];
            }
        }
        if (valid) out[(size_t)b * nt + j] = C.b ? p + C.b[j] : p;
    }
}

// MulticompartmentConnection.compute with Probability / Mask / Intensity features (topology.py:437-479,
// topology_features.py:425-429, :507-508, :755-756): conn_compute_kernel's sum over the spiking i, each term fl(w * I)
// kept only when its mask byte is set and its draw under (draw_seed, draw_step, draw_conn) transmits — the window
// gather's terms in the same order.
__global__ void __launch_bounds__(SNN_GEN_THREADS) mcc_feat_compute_kernel(snn_conn_t C, int ns, int nt, int B,
                                                                            const uint8_t *__restrict__ s, float *__restrict__ out) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int j = blockIdx.x * SNN_TILE + lane;
    const bool valid = j < nt;
    for (int b = blockIdx.y * SNN_GEN_WARPS + warp; b < B; b += gridDim.y * SNN_GEN_WARPS) {
        float p = 0.0f;
        for (int i0 = 0; i0 < ns; i0 += 32) {
            const bool sp = (i0 + lane < ns) && s[(size_t)b * ns + i0 + lane] != 0;
            uint32_t word = __ballot_sync(0xffffffffu, sp);
            while (word) {
                const int i = i0 + __ffs(word) - 1;
                word &= word - 1;
                if (!valid) continue;
                const size_t ij = (size_t)i * nt + j;
                bool keep = !C.f_mask || C.f_mask[ij] != 0;
                if (keep && C.f_prob)
                    keep = snn_synapse_transmits(snn_synapse_draw(C.draw_seed, C.draw_step, C.draw_conn, (uint32_t)i, (uint32_t)j), C.f_prob[ij]);
                if (keep) p = p + (C.f_int ? C.w[ij] * C.f_int[ij] : C.w[ij]);
            }
        }
        if (valid) out[(size_t)b * nt + j] = C.b ? p + C.b[j] : p;
    }
}

// SparseConnection.compute (topology.py:2009-2017, :332-346) on the CSR pattern: out[b,j] = the stored w[i,j] of the
// spiking i, i ascending, from +0, then the bias — the window's sparse gather without its workspace: each lane (column j)
// finds its entry of a spiking row by binary search.  Positions are clamped to [0, nnz], so a malformed pattern cannot make
// it read outside the arrays.
__global__ void __launch_bounds__(SNN_GEN_THREADS) sparse_compute_kernel(snn_conn_t C, int ns, int nt, int B,
                                                                          const uint8_t *__restrict__ s, float *__restrict__ out) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int j = blockIdx.x * SNN_TILE + lane;
    const bool valid = j < nt;
    for (int b = blockIdx.y * SNN_GEN_WARPS + warp; b < B; b += gridDim.y * SNN_GEN_WARPS) {
        float p = 0.0f;
        for (int i0 = 0; i0 < ns; i0 += 32) {
            const bool sp = (i0 + lane < ns) && s[(size_t)b * ns + i0 + lane] != 0;
            uint32_t word = __ballot_sync(0xffffffffu, sp);
            while (word) {
                const int i = i0 + __ffs(word) - 1;
                word &= word - 1;
                const int a = max(0, min(C.sp_rowptr[i], C.nnz)), e = max(a, min(C.sp_rowptr[i + 1], C.nnz));
                int lo = a, hi = e;
                while (lo < hi) {
                    const int mid = (lo + hi) >> 1;
                    if (C.sp_col[mid] < j) lo = mid + 1; else hi = mid;
                }
                if (valid && lo < e && C.sp_col[lo] == j) p = p + C.w[lo];
            }
        }
        if (valid) out[(size_t)b * nt + j] = C.b ? p + C.b[j] : p;
    }
}

__global__ void __launch_bounds__(256) scale_kernel(float *w, size_t n, float f) {
    for (size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (size_t)gridDim.x * blockDim.x) w[k] = w[k] * f;
}

// Conv2dConnection.compute (topology.py:799-815): out[b, co, oy, ox] = sum of the filter taps whose (zero-padded)
// input position spiked, in ascending (ci, ky, kx) order, then the bias — the window kernels' gather_conv on
// byte spikes.  Thread = one target neuron of one sample.
__global__ void __launch_bounds__(256) conv_compute_kernel(snn_conn_t C, int ns, int nt, int B, const uint8_t *__restrict__ s,
                                                           float *__restrict__ out) {
    const size_t total = (size_t)B * nt;
    for (size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x; k < total; k += (size_t)gridDim.x * blockDim.x) {
        const int b = (int)(k / nt), j = (int)(k - (size_t)b * nt);
        const int L = C.hout * C.wout;
        const int co = j / L, l = j - co * L, oy = l / C.wout, ox = l - oy * C.wout;
        const uint8_t *sb = s + (size_t)b * ns;
        float p = 0.0f;
        for (int ci = 0; ci < C.cin; ++ci)
            for (int ky = 0; ky < C.kh; ++ky) {
                const int iy = oy * C.sh - C.ph + ky * C.dh;
                if (iy < 0 || iy >= C.hin) continue;
                for (int kx = 0; kx < C.kw; ++kx) {
                    const int ix = ox * C.sw - C.pw + kx * C.dw;
                    if (ix < 0 || ix >= C.win) continue;
                    if (sb[(ci * C.hin + iy) * C.win + ix]) p = p + C.w[((co * C.cin + ci) * C.kh + ky) * C.kw + kx];
                }
            }
        out[k] = p + C.b[co];
    }
}

// MaxPool2dConnection / MaxPoo3dConnection.compute (topology.py:1163-1185, :1255-1277), step 1: the rates advance by
// the spikes, in place.
__global__ void __launch_bounds__(256) pool_rates_kernel(snn_conn_t C, size_t total, const uint8_t *__restrict__ s) {
    for (size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x; k < total; k += (size_t)gridDim.x * blockDim.x)
        C.pool_rates[k] = pool_rate_update(C.pool_rates[k], C.pool_decay, s[k] != 0);
}

// Steps 2-3: the spike at the window's first maximum of the updated rates (the window gather's pool_argmax; D3: the
// 3-D window); thread = one target neuron of one sample.
template <bool D3>
__global__ void __launch_bounds__(256) pool_compute_kernel(snn_conn_t C, int ns, int nt, int B, const uint8_t *__restrict__ s,
                                                           float *__restrict__ out) {
    const size_t total = (size_t)B * nt;
    for (size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x; k < total; k += (size_t)gridDim.x * blockDim.x) {
        const int b = (int)(k / nt), j = (int)(k - (size_t)b * nt);
        out[k] = s[(size_t)b * ns + pool_argmax<D3>(C, C.pool_rates + (size_t)b * ns, j)] ? 1.0f : 0.0f;
    }
}

__global__ void __launch_bounds__(SNN_GEN_THREADS) conv_normalize_kernel(snn_conn_t C, int KK) { normalize_conv_item(C, KK, blockIdx.x, gridDim.x); }

// Conv3dConnection.compute (topology.py:979-995) on byte spikes: the window gather's gather_conv3d order ((ci, kz, ky, kx)
// ascending from +0, then the bias).  Thread = one target neuron of one sample.
__global__ void __launch_bounds__(256) conv3d_compute_kernel(snn_conn_t C, int ns, int nt, int B, const uint8_t *__restrict__ s,
                                                             float *__restrict__ out) {
    const size_t total = (size_t)B * nt;
    const int HW = C.hout * C.wout, L = C.dout * HW, KK = C.kd * C.kh * C.kw;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
        const int b = (int)(e / nt), j = (int)(e - (size_t)b * nt), co = j / L, l = j - co * L;
        const int oz = l / HW, r = l - oz * HW, oy = r / C.wout, ox = r - oy * C.wout;
        const uint8_t *sb = s + (size_t)b * ns;
        const float *wf = C.w + (size_t)co * C.cin * KK;
        float p = 0.0f;
        for (int ci = 0; ci < C.cin; ++ci)
            for (int kz = 0; kz < C.kd; ++kz) {
                const int iz = oz * C.sd - C.pd + kz;
                if (iz < 0 || iz >= C.din) continue;
                for (int ky = 0; ky < C.kh; ++ky) {
                    const int iy = oy * C.sh - C.ph + ky;
                    if (iy < 0 || iy >= C.hin) continue;
                    for (int kx = 0; kx < C.kw; ++kx) {
                        const int ix = ox * C.sw - C.pw + kx;
                        if (ix < 0 || ix >= C.win) continue;
                        if (sb[((ci * C.din + iz) * C.hin + iy) * C.win + ix]) p = p + wf[((ci * C.kd + kz) * C.kh + ky) * C.kw + kx];
                    }
                }
            }
        out[e] = p + C.b[co];
    }
}

__global__ void __launch_bounds__(SNN_GEN_THREADS) conv3d_update_kernel(snn_conn_t C) { phase3_conv3d(C, blockIdx.x, gridDim.x); }

// Conv1dConnection.compute (topology.py:640-656) on byte spikes: the window gather's gather_conv1d order ((ci, kx)
// ascending from +0, then the bias).  Thread = one target neuron of one sample.
__global__ void __launch_bounds__(256) conv1d_compute_kernel(snn_conn_t C, int ns, int nt, int B, const uint8_t *__restrict__ s,
                                                             float *__restrict__ out) {
    const size_t total = (size_t)B * nt;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
        const int b = (int)(e / nt), j = (int)(e - (size_t)b * nt), co = j / C.wout, ox = j - co * C.wout;
        const uint8_t *sb = s + (size_t)b * ns;
        const float *wf = C.w + (size_t)co * C.cin * C.kw;
        float p = 0.0f;
        for (int ci = 0; ci < C.cin; ++ci)
            for (int kx = 0; kx < C.kw; ++kx) {
                const int ix = ox * C.sw - C.pw + kx;
                if (ix >= 0 && ix < C.win && sb[ci * C.win + ix]) p = p + wf[ci * C.kw + kx];
            }
        out[e] = p + C.b[co];
    }
}

__global__ void __launch_bounds__(SNN_GEN_THREADS) conv1d_update_kernel(const __grid_constant__ DevNet N, int ci) {
    phase3_conv1d(N, ci, blockIdx.x, gridDim.x, 0);
}

// LocalConnection2D.compute (topology.py:1717-1740) on byte spikes: the window gather's gather_local2d order (k ascending
// within a channel from +0, then the channels).  Thread = one target neuron of one sample.
__global__ void __launch_bounds__(256) local2d_compute_kernel(snn_conn_t C, int ns, int nt, int B, const uint8_t *__restrict__ s,
                                                              float *__restrict__ out) {
    const size_t total = (size_t)B * nt;
    const int K = C.kh * C.kw, P = C.hout * C.wout;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
        const int b = (int)(e / nt), j = (int)(e - (size_t)b * nt), l = j % P, oy = l / C.wout, ox = l - oy * C.wout;
        const uint8_t *sb = s + (size_t)b * ns;
        float p = 0.0f;
        for (int ci = 0; ci < C.cin; ++ci) {
            const float *wr = C.w + ((size_t)ci * nt + j) * K;
            float q = 0.0f;
            for (int ky = 0; ky < C.kh; ++ky)
                for (int kx = 0; kx < C.kw; ++kx)
                    if (sb[(ci * C.hin + oy * C.sh + ky) * C.win + ox * C.sw + kx]) q = q + wr[ky * C.kw + kx];
            p = p + q;
        }
        out[e] = p;
    }
}

__global__ void __launch_bounds__(SNN_GEN_THREADS) local2d_normalize_kernel(snn_conn_t C, int rows) {
    normalize_local2d_item(C, rows, C.kh * C.kw, blockIdx.x, gridDim.x);
}

__global__ void __launch_bounds__(SNN_GEN_THREADS) local2d_update_kernel(const __grid_constant__ DevNet N, int ci) {
    phase3_local2d(N, ci, blockIdx.x, gridDim.x, 0);
}

// LocalConnection3D.compute (topology.py:1866-1896) on byte spikes: the window gather's gather_local2d<.., true> order (k
// ascending within a channel from +0, then the channels).  Thread = one target neuron of one sample.
__global__ void __launch_bounds__(256) local3d_compute_kernel(snn_conn_t C, int ns, int nt, int B, const uint8_t *__restrict__ s,
                                                              float *__restrict__ out) {
    const size_t total = (size_t)B * nt;
    const int K = C.kd * C.kh * C.kw, HW = C.hout * C.wout, P = C.dout * HW;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
        const int b = (int)(e / nt), j = (int)(e - (size_t)b * nt), l = j % P, oz = l / HW, r = l - oz * HW;
        const int oy = r / C.wout, ox = r - oy * C.wout;
        const uint8_t *sb = s + (size_t)b * ns;
        float p = 0.0f;
        for (int ci = 0; ci < C.cin; ++ci) {
            const float *wr = C.w + ((size_t)ci * nt + j) * K;
            float q = 0.0f;
            for (int kz = 0; kz < C.kd; ++kz)
                for (int ky = 0; ky < C.kh; ++ky)
                    for (int kx = 0; kx < C.kw; ++kx)
                        if (sb[((ci * C.din + oz * C.sd + kz) * C.hin + oy * C.sh + ky) * C.win + ox * C.sw + kx])
                            q = q + wr[(kz * C.kh + ky) * C.kw + kx];
            p = p + q;
        }
        out[e] = p;
    }
}

__global__ void __launch_bounds__(SNN_GEN_THREADS) local3d_normalize_kernel(snn_conn_t C, int rows) {
    normalize_local2d_item(C, rows, C.kd * C.kh * C.kw, blockIdx.x, gridDim.x);
}

__global__ void __launch_bounds__(SNN_GEN_THREADS) local3d_update_kernel(const __grid_constant__ DevNet N, int ci) {
    phase3_local3d(N, ci, blockIdx.x, gridDim.x, 0);
}

// bit-pack the CURRENT spikes of the two layers of a connection into slot 0 (F32: a PassThroughNodes layer's float32 s)
template <bool F32>
__global__ void pack_bits_kernel(const uint8_t *__restrict__ s, uint32_t *__restrict__ bits, int B, int n, int nw) {
    const int lane = threadIdx.x & 31;
    const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (gw >= B * nw) return;
    const int b = gw / nw, w = gw % nw, j = w * 32 + lane;
    const bool sp = j < n && (F32 ? ((const float *)s)[(size_t)b * n + j] != 0.0f : s[(size_t)b * n + j] != 0);
    const uint32_t word = __ballot_sync(0xffffffffu, sp);
    if (lane == 0) bits[(size_t)b * nw + w] = word;
}

template <bool SYN>
__global__ void __launch_bounds__(SNN_GEN_THREADS) conn_update_kernel(const __grid_constant__ DevNet N, int ci) {
    SNN_DYN_SHARED(float, smem);
    const GenSmem M = gen_carve(smem, N.B);
    phase3<SYN>(N, ci, blockIdx.x, 0, N.layers[N.conns[ci].src].nw, 0, M);
}

// The single-operator update of an averaged MCC PostPre (snn_b200.h SNN_RULE_AVG): one step of the window's learning
// phase, a CTA per column tile; the slot bitmaps are read from a copy (DevAvg slot 1) and written to the caller's.
__global__ void __launch_bounds__(SNN_GEN_THREADS) avg_update_kernel(const __grid_constant__ DevNet N, int ci) {
    SNN_DYN_SHARED(float, smem);
    const GenSmem M = gen_carve(smem, N.B);
    phase3_mcc_avg(N, ci, blockIdx.x, 0, N.layers[N.conns[ci].src].nw, 0, M);
}
__global__ void copy_u32_kernel(uint32_t *dst, const uint32_t *src, size_t n) {
    for (size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (size_t)gridDim.x * blockDim.x) dst[k] = src[k];
}

template <bool WN>
__global__ void __launch_bounds__(SNN_GEN_THREADS) conn_normalize_kernel(snn_conn_t C, int ns, int nt) {
    SNN_SHARED(float, s_part, (SNN_NORM_CHUNKS + 1) * 32);
    normalize_tile<WN>(C, ns, nt, blockIdx.x, s_part);
}

__global__ void delta_prepare_kernel(const float *__restrict__ w, const float *__restrict__ w0, float *__restrict__ dw, size_t n) {
    for (size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (size_t)gridDim.x * blockDim.x) dw[k] = w[k] - w0[k];
}

// w = clamp(w0 + sum_r dw_r), then normalize() — all on one column tile (SURVEY.md §8e; snn_combine.cuh).
__global__ void __launch_bounds__(SNN_GEN_THREADS) delta_apply_kernel(snn_conn_t C, const float *w0, const float *__restrict__ dws, int ns, int nt,
                                                                       float *theta, const float *__restrict__ dtheta, int n_theta) {
    if (theta)   // theta = theta0 + sum_r dtheta_r, in place, spread over the grid
        for (int k = blockIdx.x * SNN_GEN_THREADS + threadIdx.x; k < n_theta; k += gridDim.x * SNN_GEN_THREADS) theta[k] = theta[k] + dtheta[k];
    SNN_SHARED(float, s_part, (SNN_NORM_CHUNKS + 1) * 32);
    delta_apply_tile(C, w0, dws, ns, nt, blockIdx.x, s_part);
}

// Checks on the device that a square matrix has the structure a plan claims for it (SNN_W_DIAG: val on the
// diagonal, 0 elsewhere; SNN_W_OFFDIAG: 0 on the diagonal, val elsewhere) — the fused kernels replace such a
// matrix by its constant, so a matrix modified behind the host-side cache must not go unnoticed.
__global__ void __launch_bounds__(256) verify_structure_kernel(const float *__restrict__ w, int n, int structure, float val, int32_t *err) {
    const size_t total = (size_t)n * n;
    const bool diag = structure == SNN_W_DIAG;
    bool bad = false;
    if ((n & 3) == 0 && (((size_t)w) & 15) == 0) {   // 16-byte loads: the matrix is read once per window (10 MB at n = 1600)
        const float4 *w4 = (const float4 *)w;
        for (size_t q = (size_t)blockIdx.x * blockDim.x + threadIdx.x; q < total / 4; q += (size_t)gridDim.x * blockDim.x) {
            const float4 x = __ldcs(w4 + q);
            const size_t k = 4 * q, i = k / n, j = k - i * n;   // 4 | n: the four elements share row i
            const float xs[4] = {x.x, x.y, x.z, x.w};
            #pragma unroll
            for (int e = 0; e < 4; ++e) bad |= xs[e] != (((i == j + e) == diag) ? val : 0.0f);
        }
    } else {
        for (size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x; k < total; k += (size_t)gridDim.x * blockDim.x) {
            const size_t i = k / n, j = k - i * n;
            bad |= w[k] != (((i == j) == diag) ? val : 0.0f);
        }
    }
    if (__syncthreads_or(bad) && threadIdx.x == 0 && err) atomicOr(err, SNN_ERR_STRUCTURE);
}

// MeanFieldConnection.compute (topology.py:1972-1981): out[b, j] = fl(fl(count / N) * w[mf_off[j] + b * mf_stride]), where
// count is the number of spikes in the whole [B, n_src] tensor and N = B * n_src (snn_b200.h).  The count couples every
// sample, so one CTA forms it (an integer: exact in any order) and then writes every output.
__global__ void __launch_bounds__(1024) meanfield_compute_kernel(snn_conn_t C, int nt, int B, int N, const uint8_t *__restrict__ s,
                                                                 float *__restrict__ out) {
    SNN_SHARED(int, s_cnt, 1);
    if (threadIdx.x == 0) s_cnt[0] = 0;
    __syncthreads();
    int c = 0;
    for (int k = threadIdx.x; k < N; k += blockDim.x) c += s[k] != 0;
    if (c) atomicAdd(s_cnt, c);
    __syncthreads();
    const float mean = (float)s_cnt[0] / (float)N;
    const size_t total = (size_t)B * nt;
    for (size_t k = threadIdx.x; k < total; k += blockDim.x) {
        const int b = (int)(k / nt), j = (int)(k - (size_t)b * nt);
        out[k] = mean * C.w[C.mf_off[j] + (size_t)b * C.mf_stride];
    }
}

inline int cuda_rc(cudaError_t e) { return e == cudaSuccess ? SNN_OK : SNN_ERR_CUDA; }

}  // namespace

int snn_verify_structure(const snn_conn_t &C, int n, int32_t *err, cudaStream_t stream) {
    if (C.structure != SNN_W_DIAG && C.structure != SNN_W_OFFDIAG) return SNN_OK;
    const size_t total = (size_t)n * n;
    const int blocks = (int)((total + 2047) / 2048 < 1184 ? (total + 2047) / 2048 : 1184);   // 8 elements per thread, up to 8 CTAs per SM
    SNN_LAUNCH(verify_structure_kernel, blocks > 0 ? blocks : 1, 256, 0, stream, C.w, n, C.structure, C.structure_val, err);
    return cuda_rc(cudaGetLastError());
}

extern "C" {

int snn_b200_conn_compute(const snn_conn_t *conn0, int32_t n_src, int32_t n_tgt, int32_t B, const uint8_t *s, float *out,
                          void *stream) {
    // the product does not read the norm (SNN_CONN_WNORM: the caller normalises after it)
    snn_conn_t K;
    if (conn0) { K = *conn0; K.kind &= ~SNN_CONN_WNORM; }
    const snn_conn_t *conn = conn0 ? &K : nullptr;
    if (!conn || (!conn->w && !(conn->kind == SNN_CONN_SPARSE && conn->nnz == 0) && !snn_is_maxpool(conn->kind)) || !s || !out ||
        n_src <= 0 || n_tgt <= 0 || B <= 0)
        return SNN_ERR_BAD_ARG;
    // (on SNN_CONN_DENSE this storage holds the per-synapse tensors, which the gather does not read)
    const bool feat = conn->kind == SNN_CONN_MCC && (conn->f_prob || conn->f_mask || conn->f_int);
    if (conn->kind != SNN_CONN_MCC && conn->kind != SNN_CONN_DENSE && (conn->f_prob || conn->f_mask || conn->f_int)) return SNN_ERR_BAD_ARG;
    if (snn_is_maxpool(conn->kind)) {   // updates conn->pool_rates [B, n_src] in place, then writes [B, n_tgt]
        const int rc = snn_pool_geometry_ok(*conn, n_src, n_tgt);
        if (rc != SNN_OK || conn->b) return rc != SNN_OK ? rc : SNN_ERR_BAD_ARG;
        const size_t total = (size_t)B * n_src, tout = (size_t)B * n_tgt;
        SNN_LAUNCH(pool_rates_kernel, (int)((total + 255) / 256 < 4736 ? (total + 255) / 256 : 4736), 256, 0, (cudaStream_t)stream, *conn, total, s);
        const int blocks = (int)((tout + 255) / 256 < 4736 ? (tout + 255) / 256 : 4736);
        if (conn->kind == SNN_CONN_MAXPOOL3D) SNN_LAUNCH(pool_compute_kernel<true>, blocks, 256, 0, (cudaStream_t)stream, *conn, n_src, n_tgt, B, s, out);
        else SNN_LAUNCH(pool_compute_kernel<false>, blocks, 256, 0, (cudaStream_t)stream, *conn, n_src, n_tgt, B, s, out);
        return cuda_rc(cudaGetLastError());
    }
    if (conn->kind == SNN_CONN_MEANFIELD) {   // the count over the batch is exact below 2^24 spikes (snn_b200.h)
        if (!conn->mf_off || conn->b || conn->mf_stride < 0 || (long long)B * n_src >= (1LL << 24)) return SNN_ERR_BAD_ARG;
        SNN_LAUNCH(meanfield_compute_kernel, 1, 1024, 0, (cudaStream_t)stream, *conn, n_tgt, B, B * n_src, s, out);
        return cuda_rc(cudaGetLastError());
    }
    if (conn->kind == SNN_CONN_LOCAL2D) {
        const int rc = snn_local2d_geometry_ok(*conn, n_src, n_tgt);
        if (rc != SNN_OK) return rc;
        const size_t total = (size_t)B * n_tgt;
        const int blocks = (int)((total + 255) / 256 < 4736 ? (total + 255) / 256 : 4736);
        SNN_LAUNCH(local2d_compute_kernel, blocks, 256, 0, (cudaStream_t)stream, *conn, n_src, n_tgt, B, s, out);
        return cuda_rc(cudaGetLastError());
    }
    if (conn->kind == SNN_CONN_LOCAL3D) {
        const int rc = snn_local3d_geometry_ok(*conn, n_src, n_tgt);
        if (rc != SNN_OK) return rc;
        const size_t total = (size_t)B * n_tgt;
        const int blocks = (int)((total + 255) / 256 < 4736 ? (total + 255) / 256 : 4736);
        SNN_LAUNCH(local3d_compute_kernel, blocks, 256, 0, (cudaStream_t)stream, *conn, n_src, n_tgt, B, s, out);
        return cuda_rc(cudaGetLastError());
    }
    if (conn->kind == SNN_CONN_CONV3D) {
        const int rc = snn_conv3d_geometry_ok(*conn, n_src, n_tgt);
        if (rc != SNN_OK) return rc;
        const size_t total = (size_t)B * n_tgt;
        const int blocks = (int)((total + 255) / 256 < 4736 ? (total + 255) / 256 : 4736);
        SNN_LAUNCH(conv3d_compute_kernel, blocks, 256, 0, (cudaStream_t)stream, *conn, n_src, n_tgt, B, s, out);
        return cuda_rc(cudaGetLastError());
    }
    if (conn->kind == SNN_CONN_CONV1D) {
        const int rc = snn_conv1d_geometry_ok(*conn, n_src, n_tgt);
        if (rc != SNN_OK) return rc;
        const size_t total = (size_t)B * n_tgt;
        const int blocks = (int)((total + 255) / 256 < 4736 ? (total + 255) / 256 : 4736);
        SNN_LAUNCH(conv1d_compute_kernel, blocks, 256, 0, (cudaStream_t)stream, *conn, n_src, n_tgt, B, s, out);
        return cuda_rc(cudaGetLastError());
    }
    if (conn->kind == SNN_CONN_CONV2D) {
        if (!conn->b || conn->cin * conn->hin * conn->win != n_src || conn->cout * conn->hout * conn->wout != n_tgt) return SNN_ERR_BAD_ARG;
        const size_t total = (size_t)B * n_tgt;
        const int blocks = (int)((total + 255) / 256 < 4736 ? (total + 255) / 256 : 4736);
        SNN_LAUNCH(conv_compute_kernel, blocks, 256, 0, (cudaStream_t)stream, *conn, n_src, n_tgt, B, s, out);
        return cuda_rc(cudaGetLastError());
    }
    dim3 grid((n_tgt + SNN_TILE - 1) / SNN_TILE, (B + SNN_GEN_WARPS - 1) / SNN_GEN_WARPS);
    if (grid.y > 64) grid.y = 64;
    if (conn->kind == SNN_CONN_SPARSE) {
        if (conn->nnz < 0 || !conn->sp_rowptr || (conn->nnz > 0 && !conn->sp_col)) return SNN_ERR_BAD_ARG;
        SNN_LAUNCH(sparse_compute_kernel, grid, SNN_GEN_THREADS, 0, (cudaStream_t)stream, *conn, n_src, n_tgt, B, s, out);
        return cuda_rc(cudaGetLastError());
    }
    if (feat) {
        SNN_LAUNCH(mcc_feat_compute_kernel, grid, SNN_GEN_THREADS, 0, (cudaStream_t)stream, *conn, n_src, n_tgt, B, s, out);
        return cuda_rc(cudaGetLastError());
    }
    SNN_LAUNCH(conn_compute_kernel, grid, SNN_GEN_THREADS, 0, (cudaStream_t)stream, *conn, n_src, n_tgt, B, s, out);
    return cuda_rc(cudaGetLastError());
}

int snn_b200_conn_update(const snn_net_t *net, int32_t ci, int32_t B, void *workspace, size_t workspace_bytes, void *stream_) {
    if (!net || ci < 0 || ci >= net->n_conns || B <= 0 || !workspace) return SNN_ERR_BAD_ARG;
    snn_conn_t C = net->conns[ci];
    if (C.kind & SNN_CONN_WNORM) {   // the norm is not the rule's (a single update is a full pass: every row is clamped)
        if (C.rule & SNN_RULE_AVG) return SNN_ERR_UNSUPPORTED;
        C.kind &= ~SNN_CONN_WNORM;
    }
    const bool avg = (C.rule & SNN_RULE_AVG) != 0;
    if (avg) {   // MCC PostPre with averaging (snn_b200.h): the plain rule's checks below, then its own kernel
        if (C.kind != SNN_CONN_MCC || (C.rule & ~SNN_RULE_AVG) != SNN_RULE_MCC_POSTPRE || C.mask) return SNN_ERR_UNSUPPORTED;
        if (C.avg_k < 1 || C.avg_idx_pre < 0 || C.avg_idx_pre >= C.avg_k || C.avg_idx_post < 0 || C.avg_idx_post >= C.avg_k ||
            !C.avg_pre || !C.avg_post || !C.avg_rows || !C.avg_cols)
            return SNN_ERR_BAD_ARG;
        C.rule = SNN_RULE_MCC_POSTPRE;
    }
    if (C.src < 0 || C.src >= net->n_layers || C.tgt < 0 || C.tgt >= net->n_layers) return SNN_ERR_BAD_ARG;
    if (C.kind == SNN_CONN_SPARSE) {   // learning.NoOp: the stored values decay (learning.py:93-94); no other rule on a fixed pattern
        if (C.rule != SNN_RULE_NONE && C.rule != SNN_RULE_NOOP) return SNN_ERR_UNSUPPORTED;
        if (C.nnz < 0 || (C.nnz > 0 && !C.w)) return SNN_ERR_BAD_ARG;
        if (C.rule == SNN_RULE_NONE || C.nnz == 0 || C.weight_decay == 0.0f || C.weight_decay == 1.0f) return SNN_OK;
        const int blocks = (int)(((size_t)C.nnz + 1023) / 1024 < 1184 ? ((size_t)C.nnz + 1023) / 1024 : 1184);
        SNN_LAUNCH(scale_kernel, blocks, 256, 0, (cudaStream_t)stream_, C.w, (size_t)C.nnz, C.weight_decay);
        return cuda_rc(cudaGetLastError());
    }
    if (!C.w) return SNN_ERR_BAD_ARG;
    if (C.kind == SNN_CONN_MEANFIELD)   // learning.NoOp scales w by 1.0 and does not clamp: nothing changes (snn_b200.h)
        return C.rule == SNN_RULE_NONE || C.rule == SNN_RULE_NOOP ? SNN_OK : SNN_ERR_UNSUPPORTED;
    if (C.kind == SNN_CONN_CONV3D) {   // decay / clamp only (snn_b200.h), dense over w
        const int rc = snn_conv3d_geometry_ok(C, net->layers[C.src].n, net->layers[C.tgt].n);
        if (rc != SNN_OK) return rc;
        if (!snn_conv3d_rule_ok(C) || C.mask) return SNN_ERR_UNSUPPORTED;
        if (C.rule == SNN_RULE_NONE) return SNN_OK;
        const size_t NW = (size_t)C.cout * C.cin * C.kd * C.kh * C.kw;
        const int blocks = (int)((NW + SNN_GEN_THREADS - 1) / SNN_GEN_THREADS < 1184 ? (NW + SNN_GEN_THREADS - 1) / SNN_GEN_THREADS : 1184);
        SNN_LAUNCH(conv3d_update_kernel, blocks, SNN_GEN_THREADS, 0, (cudaStream_t)stream_, C);
        return cuda_rc(cudaGetLastError());
    }
    const bool pass = net->layers[C.src].kind == SNN_NODE_PASSTHROUGH || net->layers[C.tgt].kind == SNN_NODE_PASSTHROUGH;
    if (pass && C.rule != SNN_RULE_NONE && C.rule != SNN_RULE_NOOP) return SNN_ERR_UNSUPPORTED;   // (snn_b200.h)
    // the single-operator update is the dense [n_src, n_tgt] rule application or a LocalConnection2D's / 3D's or
    // Conv1dConnection's; other convolutional weights and the reward-modulated rules (whose state lives in the window
    // plan) are only updated inside run_window
    const bool local = C.kind == SNN_CONN_LOCAL2D, conv1d = C.kind == SNN_CONN_CONV1D, local3d = C.kind == SNN_CONN_LOCAL3D;
    if (C.kind != SNN_CONN_DENSE && C.kind != SNN_CONN_MCC && !local && !conv1d && !local3d) return SNN_ERR_UNSUPPORTED;
    if (local3d) {
        const int rc = snn_local3d_geometry_ok(C, net->layers[C.src].n, net->layers[C.tgt].n);
        if (rc != SNN_OK) return rc;
        if (!snn_local_rule_ok(C) || C.mask) return SNN_ERR_UNSUPPORTED;
    }
    if (local) {
        const int rc = snn_local2d_geometry_ok(C, net->layers[C.src].n, net->layers[C.tgt].n);
        if (rc != SNN_OK) return rc;
        if (C.rule == SNN_RULE_MCC_POSTPRE) return SNN_ERR_UNSUPPORTED;
    }
    if (conv1d) {
        const int rc = snn_conv1d_geometry_ok(C, net->layers[C.src].n, net->layers[C.tgt].n);
        if (rc != SNN_OK) return rc;
        if (!snn_conv1d_rule_ok(C) || C.mask) return SNN_ERR_UNSUPPORTED;
    }
    if (SNN_RULE_IS_MSTDP(C.rule)) return SNN_ERR_UNSUPPORTED;
    const bool syn = snn_has_syn(C);
    if (syn) {
        const int rc = snn_syn_check(C);
        if (rc != SNN_OK) return rc;
    }
    if (C.rule == SNN_RULE_NONE) return SNN_OK;
    cudaStream_t stream = (cudaStream_t)stream_;
    DevNet N;
    memset(&N, 0, sizeof(N));
    N.n_layers = net->n_layers; N.n_conns = net->n_conns; N.learning = 1; N.T = 1; N.B = B;
    for (int c = 0; c < net->n_conns; ++c) N.conns[c] = net->conns[c];
    N.conns[ci] = C;
    size_t off = 0;
    const int ends[2] = {C.src, C.tgt};
    for (int e = 0; e < 2; ++e) {
        const int l = ends[e];
        DevLayer &D = N.layers[l];
        if (D.bits) continue;  // recurrent connection: same layer twice
        D.L = net->layers[l];
        D.nw = (D.L.n + 31) / 32;
        D.bits = (uint32_t *)((char *)workspace + off);
        off += (sizeof(uint32_t) * (size_t)B * D.nw + 255) / 256 * 256;
        D.xpub = D.L.x;  // slot 0 = the layer's current trace
        if (off > workspace_bytes) return SNN_ERR_WORKSPACE;
        const int warps = B * D.nw;
        if (D.L.kind == SNN_NODE_PASSTHROUGH) SNN_LAUNCH(pack_bits_kernel<true>, (warps * 32 + 255) / 256, 256, 0, stream, D.L.s, D.bits, B, D.L.n, D.nw);
        else SNN_LAUNCH(pack_bits_kernel<false>, (warps * 32 + 255) / 256, 256, 0, stream, D.L.s, D.bits, B, D.L.n, D.nw);
    }
    if (local) {   // dense over w, spread over the grid like the window's learning phase
        const size_t NW = (size_t)N.layers[C.tgt].L.n * C.cin * C.kh * C.kw;
        const int blocks = (int)((NW + SNN_GEN_THREADS - 1) / SNN_GEN_THREADS < 1184 ? (NW + SNN_GEN_THREADS - 1) / SNN_GEN_THREADS : 1184);
        SNN_LAUNCH(local2d_update_kernel, blocks, SNN_GEN_THREADS, 0, stream, N, ci);
        return cuda_rc(cudaGetLastError());
    }
    if (local3d) {   // one warp per row segment, like the window's learning phase
        const size_t units = (size_t)N.layers[C.tgt].L.n * ((C.cin * C.kd * C.kh * C.kw + 32 * SNN_LOCAL3D_EPL - 1) / (32 * SNN_LOCAL3D_EPL));
        const int blocks = (int)((units + SNN_GEN_WARPS - 1) / SNN_GEN_WARPS < 1184 ? (units + SNN_GEN_WARPS - 1) / SNN_GEN_WARPS : 1184);
        SNN_LAUNCH(local3d_update_kernel, blocks, SNN_GEN_THREADS, 0, stream, N, ci);
        return cuda_rc(cudaGetLastError());
    }
    if (conv1d) {   // one warp per group of elements, like the window's learning phase
        const size_t NW = (size_t)C.cout * C.cin * C.kw;
        const int blocks = (int)((NW + SNN_GEN_WARPS - 1) / SNN_GEN_WARPS < 1184 ? (NW + SNN_GEN_WARPS - 1) / SNN_GEN_WARPS : 1184);
        SNN_LAUNCH(conv1d_update_kernel, blocks, SNN_GEN_THREADS, 0, stream, N, ci);
        return cuda_rc(cudaGetLastError());
    }
    const size_t smem = gen_smem_bytes(B);
    if (avg) {   // the bitmaps this step reads: a copy of the caller's (the kernel rewrites them while other CTAs read)
        const size_t nr = (size_t)C.avg_k * N.layers[C.src].nw, nc = (size_t)C.avg_k * N.layers[C.tgt].nw;
        DevAvg &A = N.avg[ci];
        A.rows[0] = C.avg_rows; A.cols[0] = C.avg_cols;
        A.rows[1] = (uint32_t *)((char *)workspace + off);
        off += (sizeof(uint32_t) * nr + 255) / 256 * 256;
        A.cols[1] = (uint32_t *)((char *)workspace + off);
        off += (sizeof(uint32_t) * nc + 255) / 256 * 256;
        if (off > workspace_bytes) return SNN_ERR_WORKSPACE;
        SNN_LAUNCH(copy_u32_kernel, 1, 256, 0, stream, A.rows[1], (const uint32_t *)C.avg_rows, nr);
        SNN_LAUNCH(copy_u32_kernel, 1, 256, 0, stream, A.cols[1], (const uint32_t *)C.avg_cols, nc);
        cudaFuncSetAttribute(avg_update_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        SNN_LAUNCH(avg_update_kernel, N.layers[C.tgt].nw, SNN_GEN_THREADS, smem, stream, N, ci);
        return cuda_rc(cudaGetLastError());
    }
    if (syn) {
        cudaFuncSetAttribute(conn_update_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        SNN_LAUNCH(conn_update_kernel<true>, N.layers[C.tgt].nw, SNN_GEN_THREADS, smem, stream, N, ci);
    } else {
        cudaFuncSetAttribute(conn_update_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        SNN_LAUNCH(conn_update_kernel<false>, N.layers[C.tgt].nw, SNN_GEN_THREADS, smem, stream, N, ci);
    }
    return cuda_rc(cudaGetLastError());
}

int snn_b200_conn_normalize(const snn_conn_t *conn, int32_t n_src, int32_t n_tgt, void *stream) {
    if (!conn || n_src <= 0 || n_tgt <= 0) return SNN_ERR_BAD_ARG;
    if (conn->kind & SNN_CONN_WNORM) {   // a norm tensor, or the per-step formula when norm_step is set (snn_b200.h)
        const int kind = conn->kind & ~SNN_CONN_WNORM;
        if (kind != SNN_CONN_DENSE && kind != SNN_CONN_MCC) return SNN_ERR_UNSUPPORTED;
        if (!conn->w || (conn->norm_step != 0 && conn->norm_step != 1)) return SNN_ERR_BAD_ARG;
        if (!conn->has_norm) return SNN_OK;
        SNN_LAUNCH(conn_normalize_kernel<true>, (n_tgt + SNN_TILE - 1) / SNN_TILE, SNN_GEN_THREADS, 0, (cudaStream_t)stream, *conn, n_src, n_tgt);
        return cuda_rc(cudaGetLastError());
    }
    // the reference's normalize fails on a sparse w, and on a mean-field one with norm set
    if (conn->kind == SNN_CONN_SPARSE || (conn->kind == SNN_CONN_MEANFIELD && conn->has_norm)) return SNN_ERR_UNSUPPORTED;
    if (!conn->w) return SNN_ERR_BAD_ARG;
    if (!conn->has_norm) return SNN_OK;
    if (conn->kind == SNN_CONN_LOCAL2D) {   // rows of w viewed as [cin * n_tgt, K]
        const int rows = conn->cin * n_tgt;
        SNN_LAUNCH(local2d_normalize_kernel, (rows + SNN_GEN_THREADS - 1) / SNN_GEN_THREADS, SNN_GEN_THREADS, 0, (cudaStream_t)stream, *conn, rows);
        return cuda_rc(cudaGetLastError());
    }
    if (conn->kind == SNN_CONN_LOCAL3D) {   // rows of w viewed as [cin * n_tgt, K]
        const int rows = conn->cin * n_tgt;
        SNN_LAUNCH(local3d_normalize_kernel, (rows + SNN_GEN_THREADS - 1) / SNN_GEN_THREADS, SNN_GEN_THREADS, 0, (cudaStream_t)stream, *conn, rows);
        return cuda_rc(cudaGetLastError());
    }
    if (conn->kind == SNN_CONN_CONV2D) {
        const int F = conn->cout * conn->cin;
        SNN_LAUNCH(conv_normalize_kernel, (F + SNN_GEN_THREADS - 1) / SNN_GEN_THREADS, SNN_GEN_THREADS, 0, (cudaStream_t)stream, *conn, conn->kh * conn->kw);
        return cuda_rc(cudaGetLastError());
    }
    if (conn->kind == SNN_CONN_CONV3D) {   // rows of w viewed as [cout * cin, kd * kh * kw]
        const int F = conn->cout * conn->cin;
        SNN_LAUNCH(conv_normalize_kernel, (F + SNN_GEN_THREADS - 1) / SNN_GEN_THREADS, SNN_GEN_THREADS, 0, (cudaStream_t)stream, *conn,
                   conn->kd * conn->kh * conn->kw);
        return cuda_rc(cudaGetLastError());
    }
    if (conn->kind == SNN_CONN_CONV1D) {   // rows of w viewed as [cout * cin, kw]
        const int F = conn->cout * conn->cin;
        SNN_LAUNCH(conv_normalize_kernel, (F + SNN_GEN_THREADS - 1) / SNN_GEN_THREADS, SNN_GEN_THREADS, 0, (cudaStream_t)stream, *conn, conn->kw);
        return cuda_rc(cudaGetLastError());
    }
    SNN_LAUNCH(conn_normalize_kernel<false>, (n_tgt + SNN_TILE - 1) / SNN_TILE, SNN_GEN_THREADS, 0, (cudaStream_t)stream, *conn, n_src, n_tgt);
    return cuda_rc(cudaGetLastError());
}

int snn_b200_delta_prepare(const float *w, const float *w0, float *dw, size_t count, void *stream) {
    if (!w || !w0 || !dw) return SNN_ERR_BAD_ARG;
    const int blocks = (int)((count + 1023) / 1024 < 1184 ? (count + 1023) / 1024 : 1184);
    SNN_LAUNCH(delta_prepare_kernel, blocks > 0 ? blocks : 1, 256, 0, (cudaStream_t)stream, w, w0, dw, count);
    return cuda_rc(cudaGetLastError());
}

int snn_b200_delta_apply(float *w, const float *w0, const float *dw_sum, int32_t n_src, int32_t n_tgt, int32_t has_clamp,
                         float wmin, float wmax, int32_t has_norm, int32_t norm_abs, float norm, void *stream) {
    if (!w || !w0 || !dw_sum || n_src <= 0 || n_tgt <= 0) return SNN_ERR_BAD_ARG;
    snn_conn_t C;
    memset(&C, 0, sizeof(C));
    C.w = w; C.has_clamp = has_clamp; C.wmin = wmin; C.wmax = wmax; C.has_norm = has_norm; C.norm_abs = norm_abs; C.norm = norm;
    SNN_LAUNCH(delta_apply_kernel, (n_tgt + SNN_TILE - 1) / SNN_TILE, SNN_GEN_THREADS, 0, (cudaStream_t)stream, C, w0, dw_sum, n_src, n_tgt, nullptr, nullptr, 0);
    return cuda_rc(cudaGetLastError());
}

int snn_b200_delta_apply_fused(float *w, const float *dw_sum, int32_t n_src, int32_t n_tgt, int32_t has_clamp, float wmin, float wmax,
                               int32_t has_norm, int32_t norm_abs, float norm, float *theta, const float *dtheta_sum, int32_t n_theta,
                               void *stream) {
    if (!w || !dw_sum || n_src <= 0 || n_tgt <= 0 || (theta && (!dtheta_sum || n_theta <= 0))) return SNN_ERR_BAD_ARG;
    snn_conn_t C;
    memset(&C, 0, sizeof(C));
    C.w = w; C.has_clamp = has_clamp; C.wmin = wmin; C.wmax = wmax; C.has_norm = has_norm; C.norm_abs = norm_abs; C.norm = norm;
    SNN_LAUNCH(delta_apply_kernel, (n_tgt + SNN_TILE - 1) / SNN_TILE, SNN_GEN_THREADS, 0, (cudaStream_t)stream, C, w, dw_sum, n_src, n_tgt, theta, dtheta_sum,
                                                                                                        n_theta);
    return cuda_rc(cudaGetLastError());
}

}  // extern "C"
