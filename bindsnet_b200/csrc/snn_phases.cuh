// snn_phases.cuh — the per-step building blocks of the window kernels (spike gather, neuron
// update, one_spike resolution, STDP tile update, column normalisation), shared by the generic
// window kernel (snn_generic.cu) and the single-operator entry points (snn_ops.cu).
#pragma once
#include "snn_common.cuh"

namespace {

// ---------------------------------------------------------------------------------------
// Shared memory of one CTA of the generic tier (dynamic; carved the same way by the window kernel and by
// the single-operator kernels).  Phases never overlap inside a CTA, so the regions are reused:
//   acc     phase 3: per-warp [32 rows][32 columns] pre-synaptic accumulators (32 KB)
//           phase 1: the per-warp spike lists of the gather (first 16 KB) and the staged source bit rows of a
//                    convolutional gather (second 16 KB)
//   xs      phase 3: per-warp staged pre-synaptic traces of the samples with a post-synaptic event (16 KB)
//           phase 1: staged filter taps of a convolutional gather
//           phase 3 (conv MSTDP): the sample's two bit rows, its decoded source-spike list, the channel offsets
//   xt      phase 3: the target traces of the whole tile [B][32]; phase 3 (dense MSTDP): staged rule state
//   acc     phase 3 (conv MSTDP) also: the P- rows of the unit's output channels
#define SNN_P3_MAXEV 16
#define SNN_GATHER_BLOCK 1024   // source neurons per gather block (32 words): list capacity per warp
#define SNN_CONV_STAGE_WORDS 4096   // staged source bit words of a conv gather (second half of acc)
#define SNN_CONV_STAGE_TAPS 4096    // staged filter taps (xs region)
#define SNN_XT_MAX_BYTES (96 * 1024)

struct GenSmem {
    float *acc;
    uint16_t *list;     // [WARPS][SNN_GATHER_BLOCK]  (aliases acc)
    uint32_t *cbits;    // [SNN_CONV_STAGE_WORDS]     (aliases acc + 16 KB)
    float *red;         // [SNN_NORM_CHUNKS + 1][32]
    uint32_t *colmask;  // [ceil(B/32)][32]
    float *xs;          // [WARPS][SNN_P3_MAXEV][32]
    int32_t *evb;       // [SNN_P3_MAXEV + 1]
    uint8_t *evslot;    // [B]
    float *xt;          // [B][32] or NULL (batch too large to stage)
    uint32_t *live;     // [ceil(B/32)] samples whose staged trace row is not all zero
    int32_t xt_bytes;
};

__host__ __device__ inline size_t gen_xt_bytes(int B) {
    const size_t b = sizeof(float) * 32 * (size_t)B;
    return b <= SNN_XT_MAX_BYTES ? b : 0;
}
__host__ __device__ inline size_t gen_smem_bytes(int B) {
    const size_t NG = (size_t)((B + 31) / 32);
    size_t s = sizeof(float) * SNN_GEN_WARPS * 32 * 32;            // acc
    s += sizeof(float) * (SNN_NORM_CHUNKS + 1) * 32;               // red
    s += sizeof(uint32_t) * 32 * NG;                               // colmask
    s += sizeof(float) * SNN_GEN_WARPS * SNN_P3_MAXEV * 32;        // xs
    s += sizeof(int32_t) * (SNN_P3_MAXEV + 16);                    // evb (padded)
    s += ((size_t)B + 15) / 16 * 16;                               // evslot
    s += (sizeof(uint32_t) * NG + 15) / 16 * 16;                   // live
    s += gen_xt_bytes(B);
    return s;
}
__device__ __forceinline__ GenSmem gen_carve(float *smem, int B) {
    GenSmem M;
    const int NG = (B + 31) / 32;
    M.acc = smem;
    M.list = (uint16_t *)smem;
    M.cbits = (uint32_t *)(smem + SNN_GEN_WARPS * 32 * 16);
    M.red = smem + SNN_GEN_WARPS * 32 * 32;
    M.colmask = (uint32_t *)(M.red + (SNN_NORM_CHUNKS + 1) * 32);
    M.xs = (float *)(M.colmask + 32 * NG);
    M.evb = (int32_t *)(M.xs + SNN_GEN_WARPS * SNN_P3_MAXEV * 32);
    M.evslot = (uint8_t *)(M.evb + SNN_P3_MAXEV + 16);
    M.live = (uint32_t *)(M.evslot + (B + 15) / 16 * 16);
    M.xt_bytes = (int32_t)gen_xt_bytes(B);
    M.xt = M.xt_bytes ? (float *)((uint8_t *)M.live + (sizeof(uint32_t) * NG + 15) / 16 * 16) : nullptr;
    return M;
}

__device__ __forceinline__ float ld_ext(const snn_layer_t &L, size_t idx, bool &nonbin) {
    if (L.ext_dtype == SNN_EXT_U8) {
        const uint8_t e = ((const uint8_t *)L.ext)[idx];
        nonbin |= e > 1;
        return (float)e;
    }
    const float e = ((const float *)L.ext)[idx];
    nonbin |= (e != 0.0f && e != 1.0f);
    return e;
}

// Spike-gather for one sample: p[j] = sum_{i : s_src[b,i]} w[i, j], i ascending.
// Restates Connection.compute (topology.py:332-346) and MulticompartmentConnection.compute
// with a Weight feature (topology.py:437-479, topology_features.py:633-645) without ever
// materialising the [B, n_src, n_tgt] broadcast.  Per block of 32 words (1024 source neurons) the warp
// first compacts the set bits into an ascending index list in shared memory (ballot-free prefix sum of
// the lanes' popcounts), then walks the list eight entries at a time so that eight weight rows are in
// flight from L2 at once — the sum itself stays one fp32 add per spike in ascending i, like the oracle.
// Weights are read with ld.cg: the CTA that updates a tile in the learning phase is not the CTA that
// gathers from it.
// `first` = the lane's word of block 0 (sb[lane]), loaded by the caller ahead of time.  The words of up to eight
// blocks (8192 source neurons) are fetched together, so a wide but sparse source layer (the 6400 inhibitory neurons of
// BASELINE config 3: 7 blocks, almost always empty) costs one L2 round trip instead of one per block.
// FEAT: the connection may carry the MCC features f_prob / f_mask / f_int (snn_b200.h).  A visited synapse then adds
// fl(w * I) only when its mask byte is set and its draw under (seed, step, conn) transmits; the Probability and Mask
// factors are exact 0 / 1 in the reference, so dropping those terms leaves the reference's sum.  With FEAT = false the
// function is the plain gather.
template <bool FEAT>
__device__ __forceinline__ float gather(const snn_conn_t &C, const uint32_t *__restrict__ sb, int nw_src,
                                        int n_src, int n_tgt, int j, bool valid, int lane, uint16_t *__restrict__ lst, uint32_t first,
                                        uint32_t seed = 0u, uint32_t step = 0u, uint32_t conn = 0u) {
    float p = 0.0f;
    const float *__restrict__ wcol = C.w + j;
    for (int s0 = 0; s0 < nw_src; s0 += 256) {
        uint32_t wd[8];
        #pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int w = s0 + 32 * k + lane;
            wd[k] = (k == 0 && s0 == 0) ? first : (w < nw_src ? __ldcg(sb + w) : 0u);
        }
        uint32_t nzb = 0;   // blocks of this group that hold a spike
        #pragma unroll
        for (int k = 0; k < 8; ++k) nzb |= __any_sync(0xffffffffu, wd[k] != 0u) ? (1u << k) : 0u;
        while (nzb) {
            const int kb = __ffs(nzb) - 1;
            nzb &= nzb - 1;
            uint32_t mine = wd[0];
            #pragma unroll
            for (int k = 1; k < 8; ++k)
                if (kb == k) mine = wd[k];
            const int cnt = __popc(mine);
            int pre = cnt;
            #pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int v = __shfl_up_sync(0xffffffffu, pre, o);
                if (lane >= o) pre += v;
            }
            const int total = __shfl_sync(0xffffffffu, pre, 31);
            int q = pre - cnt;
            while (mine) {
                const int r = __ffs(mine) - 1;
                mine &= mine - 1;
                lst[q++] = (uint16_t)((lane << 5) | r);
            }
            __syncwarp();
            const int base = (s0 + 32 * kb) * 32;
            for (int e = 0; e < total; e += 8) {
                float v[8];
                #pragma unroll
                for (int k = 0; k < 8; ++k) {
                    const int i = base + (int)lst[min(e + k, total - 1)];
                    v[k] = (valid && e + k < total && i < n_src) ? __ldcg(wcol + (size_t)i * n_tgt) : 0.0f;
                }
                if (FEAT) {
                    float pr[8], in[8];
                    uint8_t mk[8];
                    #pragma unroll
                    for (int k = 0; k < 8; ++k) {
                        const int i = base + (int)lst[min(e + k, total - 1)];
                        const bool ok = valid && e + k < total && i < n_src;
                        const size_t ij = (size_t)i * n_tgt + j;
                        pr[k] = (ok && C.f_prob) ? __ldcg(C.f_prob + ij) : 1.0f;
                        mk[k] = (ok && C.f_mask) ? __ldcg(C.f_mask + ij) : (uint8_t)1;
                        in[k] = (ok && C.f_int) ? __ldcg(C.f_int + ij) : 1.0f;
                    }
                    #pragma unroll
                    for (int k = 0; k < 8; ++k) {
                        const int i = base + (int)lst[min(e + k, total - 1)];
                        bool keep = mk[k] != 0;
                        if (C.f_prob) keep = keep && snn_synapse_transmits(snn_synapse_draw(seed, step, conn, (uint32_t)i, (uint32_t)j), pr[k]);
                        if (C.f_int) v[k] = v[k] * in[k];
                        if (!keep) v[k] = 0.0f;
                    }
                }
                #pragma unroll
                for (int k = 0; k < 8; ++k)
                    if (e + k < total) p = p + v[k];
            }
            __syncwarp();
        }
    }
    return p;
}

// ---------------------------------------------------------------------------------------
// SparseConnection (SNN_CONN_SPARSE, topology.py:2009-2017).  Both functions run alone between grid barriers and are
// kept out of line, so that the register allocation of the rest of the window kernel does not depend on them.
//
// Window pre-pass: the column-block offset table of connection `c` (DevSparse::off), one warp per source row, rows spread
// over every warp of the grid.  The pattern is checked on the way: a row whose rowptr is out of [0, nnz] or not monotone,
// or whose columns are out of range or not strictly ascending, raises SNN_ERR_BAD_ARG and is entered as an empty row, so
// that the gather never reads outside the arrays.
__device__ __noinline__ void sparse_prepass(const DevNet &N, int c, int gwarp, int nwarps) {
    const snn_conn_t &C = N.conns[c];
    const DevSparse &P = N.sp[c];
    const int ns = N.layers[C.src].L.n, nt = N.layers[C.tgt].L.n, nb = P.nb, bw = P.bw;
    const int lane = threadIdx.x & 31;
    const int32_t *__restrict__ col = C.sp_col;
    for (int i = gwarp; i < ns; i += nwarps) {
        const int a = __ldg(C.sp_rowptr + i), e = __ldg(C.sp_rowptr + i + 1);
        bool bad = a < 0 || e < a || e > C.nnz;
        if (!bad)
            for (int p = a + lane; p < e; p += 32) {
                const int cj = __ldg(col + p);
                bad |= cj < 0 || cj >= nt || (p > a && cj <= __ldg(col + p - 1));
            }
        int32_t *o = P.off + (size_t)i * (nb + 1);
        if (__any_sync(0xffffffffu, bad)) {
            for (int k = lane; k <= nb; k += 32) o[k] = 0;
            if (lane == 0 && N.err) atomicOr(N.err, SNN_ERR_BAD_ARG);
            continue;
        }
        // o[k] = first position of the row with column >= k * bw: every k is written by exactly one lane
        for (int p = a + lane; p < e; p += 32) {
            const int kb = __ldg(col + p) / bw, kp = p > a ? __ldg(col + p - 1) / bw : -1;
            for (int k = kp + 1; k <= kb; ++k) o[k] = p;
        }
        const int kl = e > a ? __ldg(col + e - 1) / bw : -1;
        for (int k = kl + 1 + lane; k <= nb; k += 32) o[k] = e;
    }
}

// Sparse gather, unit = (connection, column block, chunk of SNN_GEN_WARPS samples); warp w takes sample chunk * 8 + w.
// The block's sums live in the warp's slice of the accumulator region (bw <= 1024 floats).  The warp compacts the
// sample's spiking sources into an ascending list (1024 at a time, as the dense gather does), fetches the block segments
// of 32 listed rows at once (one row per lane), then walks the rows in ascending order, eight rows' first 32 entries in
// flight together; the lanes of a row touch distinct columns and a __syncwarp separates consecutive rows, so every
// column is summed in ascending i from +0 — the dense gather's sum without its zero terms.  `cur`: the source's spikes
// of this step (one-step mode) instead of the previous one.
#define SNN_SPARSE_ROWS 8
__device__ __noinline__ void phase_sparse(const DevNet &N, int c, int blk, int chunk, bool cur, int t, const GenSmem &M) {
    const snn_conn_t &C = N.conns[c];
    const DevSparse &P = N.sp[c];
    const DevLayer &S = N.layers[C.src];
    const int B = N.B, nt = N.layers[C.tgt].L.n, nb = P.nb, bw = P.bw;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int b = chunk * SNN_GEN_WARPS + warp;
    if (b >= B) return;
    const int j0 = blk * bw, jn = min(bw, nt - j0);
    float *acc = M.acc + warp * SNN_GATHER_BLOCK;
    uint16_t *lst = (uint16_t *)M.xs + warp * SNN_GATHER_BLOCK;
    for (int x = lane; x < bw; x += 32) acc[x] = 0.0f;
    __syncwarp();
    const int slot = cur ? (t & 1) : ((t + 1) & 1);
    const bool any = !S.anyf || __ldcg(S.anyf + (size_t)(cur ? t % 3 : (t + 2) % 3) * B + b) != 0u;
    const int32_t *__restrict__ col = C.sp_col;
    const float *__restrict__ wv = C.w;
    const int32_t *__restrict__ offb = P.off + blk;
    const uint32_t *sb = S.bits + ((size_t)slot * B + b) * S.nw;
    for (int w0 = 0; any && w0 < S.nw; w0 += 32) {
        uint32_t mine = w0 + lane < S.nw ? __ldcg(sb + w0 + lane) : 0u;
        if (!__any_sync(0xffffffffu, mine != 0u)) continue;
        const int cnt = __popc(mine);
        int pre = cnt;
        #pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, pre, o);
            if (lane >= o) pre += v;
        }
        const int total = __shfl_sync(0xffffffffu, pre, 31);
        int q = pre - cnt;
        while (mine) {
            const int r = __ffs(mine) - 1;
            mine &= mine - 1;
            lst[q++] = (uint16_t)((lane << 5) | r);
        }
        __syncwarp();
        const size_t base = (size_t)w0 * 32;
        for (int e0 = 0; e0 < total; e0 += 32) {
            const int nr = min(32, total - e0);
            int p0 = 0, p1 = 0;   // segment of my row in this block
            if (lane < nr) {
                const int32_t *o = offb + (base + lst[e0 + lane]) * (size_t)(nb + 1);
                p0 = __ldcg(o);
                p1 = __ldcg(o + 1);
            }
            for (int r0 = 0; r0 < nr; r0 += SNN_SPARSE_ROWS) {
                int a[SNN_SPARSE_ROWS], e[SNN_SPARSE_ROWS], cj[SNN_SPARSE_ROWS];
                float v[SNN_SPARSE_ROWS];
                #pragma unroll
                for (int k = 0; k < SNN_SPARSE_ROWS; ++k) {
                    a[k] = __shfl_sync(0xffffffffu, p0, (r0 + k) & 31);
                    e[k] = __shfl_sync(0xffffffffu, p1, (r0 + k) & 31);
                    if (r0 + k >= nr) e[k] = a[k];
                    const bool ok = a[k] + lane < e[k];
                    cj[k] = ok ? __ldg(col + a[k] + lane) : j0;
                    v[k] = ok ? __ldcg(wv + a[k] + lane) : 0.0f;
                }
                #pragma unroll
                for (int k = 0; k < SNN_SPARSE_ROWS; ++k) {
                    if (a[k] + lane < e[k]) acc[cj[k] - j0] = acc[cj[k] - j0] + v[k];
                    for (int p = a[k] + 32 + lane; p < e[k]; p += 32) {   // rows with more than 32 entries in the block
                        const int jj = __ldg(col + p) - j0;
                        acc[jj] = acc[jj] + __ldcg(wv + p);
                    }
                    __syncwarp();
                }
            }
        }
        __syncwarp();   // the list is rewritten by the next group of words
    }
    __syncwarp();
    for (int x = lane; x < jn; x += 32) P.out[(size_t)b * nt + j0 + x] = acc[x];
    __syncwarp();   // the accumulator belongs to the warp's next unit
}

// Conv2dConnection.compute (topology.py:799-815) for one target neuron j = (co, oy, ox) of one
// sample: the sum of the filter taps whose (zero-padded) input position spiked, in ascending
// (ci, ky, kx) order, then the bias.  STAGED: the sample's source bit row and the filter taps of the
// tile's output channels sit in shared memory (phase 1 stages them once per work unit).
// The part of the gather that depends on the target neuron only (not on the sample): computed once per work unit.
struct ConvGeo {
    int co;                // output channel of neuron j
    int y0, x0;            // source row of filter row 0 (oy*sh - ph); source column of the first VALID tap of a filter row
    int kx_lo, cnt;        // first valid tap of a filter row, number of valid taps
    int ky_lo, ky_hi;      // valid filter rows (source row inside the image)
};
__device__ __forceinline__ ConvGeo conv_geo(const snn_conn_t &C, int j, bool valid) {
    ConvGeo g;
    const int L = C.hout * C.wout;
    g.co = valid ? j / L : 0;
    const int l = valid ? j - g.co * L : 0;
    const int oy = l / C.wout, ox = l - oy * C.wout;
    const int ix0 = ox * C.sw - C.pw;
    g.kx_lo = max(0, -ix0);
    g.x0 = ix0 + g.kx_lo;
    g.cnt = min(C.kw, C.win - ix0) - g.kx_lo;
    // rows: iy = y0 + ky*dh in [0, hin)
    g.y0 = oy * C.sh - C.ph;
    g.ky_lo = g.y0 < 0 ? (-g.y0 + C.dh - 1) / C.dh : 0;
    g.ky_hi = min(C.kh, g.y0 >= C.hin ? 0 : (C.hin - 1 - g.y0) / C.dh + 1);
    return g;
}

template <bool STAGED_BITS, bool STAGED_TAPS>
__device__ __forceinline__ float gather_conv(const snn_conn_t &C, const uint32_t *sb, const float *taps, int co_base, int j, bool valid,
                                             const ConvGeo &g) {
    if (!valid) return 0.0f;
    const int co = g.co;
    const int KK = C.kh * C.kw;
    float p = 0.0f;
    if (C.dw == 1 && C.kw <= 32) {
        // the kw taps of one filter row look at kw CONSECUTIVE source bits: cut that window out of the bit row (two
        // words, one funnel shift) and visit its set bits only — ascending kx, so the order of the sum is unchanged
        if (g.cnt > 0) {
            const float *tp = STAGED_TAPS ? taps + (co - co_base) * C.cin * KK : C.w + (size_t)co * C.cin * KK;
            const uint32_t cmask = g.cnt >= 32 ? 0xffffffffu : ((1u << g.cnt) - 1u);
            for (int ci = 0; ci < C.cin; ++ci)
                for (int ky = g.ky_lo; ky < g.ky_hi; ++ky) {
                    const int iy = g.y0 + ky * C.dh;
                    const int bit0 = (ci * C.hin + iy) * C.win + g.x0, w0 = bit0 >> 5, sft = bit0 & 31;
                    const uint32_t lo = STAGED_BITS ? sb[w0] : __ldcg(sb + w0);
                    const uint32_t hi = sft + g.cnt > 32 ? (STAGED_BITS ? sb[w0 + 1] : __ldcg(sb + w0 + 1)) : 0u;
                    uint32_t bits = __funnelshift_r(lo, hi, sft) & cmask;
                    const int k0 = (ci * C.kh + ky) * C.kw + g.kx_lo;
                    while (bits) {
                        const int k = k0 + __ffs(bits) - 1;
                        bits &= bits - 1;
                        p = p + (STAGED_TAPS ? tp[k] : __ldcg(tp + k));
                    }
                }
        }
        return p + C.b[co];
    }
    const int L = C.hout * C.wout, l = j - co * L, oy = l / C.wout, ox = l - oy * C.wout;   // dilated columns: tap by tap
    for (int ci = 0; ci < C.cin; ++ci)
        for (int ky = 0; ky < C.kh; ++ky) {
            const int iy = oy * C.sh - C.ph + ky * C.dh;
            if (iy < 0 || iy >= C.hin) continue;
            for (int kx = 0; kx < C.kw; ++kx) {
                const int ix = ox * C.sw - C.pw + kx * C.dw;
                if (ix < 0 || ix >= C.win) continue;
                const int i = (ci * C.hin + iy) * C.win + ix;
                const uint32_t word = STAGED_BITS ? sb[i >> 5] : __ldcg(sb + (i >> 5));
                if ((word >> (i & 31)) & 1u) {
                    const int k = (ci * C.kh + ky) * C.kw + kx;
                    p = p + (STAGED_TAPS ? taps[(co - co_base) * C.cin * KK + k] : __ldcg(C.w + (size_t)co * C.cin * KK + k));
                }
            }
        }
    return p + C.b[co];
}

// Conv3dConnection.compute (topology.py:979-995) for one target neuron j = (co, oz, oy, ox) of one sample: the sum of the
// filter taps whose (zero-padded) input position spiked, in ascending (ci, kz, ky, kx) order from +0, then the bias
// (gather_conv's order with a depth loop).  The valid taps of a kernel row look at consecutive source bits: each run of
// up to 32 is cut out of the bit row with one funnel shift and only its set bits are visited.  STAGED_BITS / STAGED_TAPS:
// the sample's source bit row / the taps of the tile's output channels sit in shared memory (staged by phase 1).
template <bool STAGED_BITS, bool STAGED_TAPS>
__device__ __forceinline__ float gather_conv3d(const snn_conn_t &C, const uint32_t *sb, const float *taps, int co_base, int j, bool valid) {
    if (!valid) return 0.0f;
    const int HW = C.hout * C.wout, L = C.dout * HW, co = j / L, l = j - co * L;
    const int oz = l / HW, r = l - oz * HW, oy = r / C.wout, ox = r - oy * C.wout;
    const int iz0 = oz * C.sd - C.pd, iy0 = oy * C.sh - C.ph, ix0 = ox * C.sw - C.pw;
    const int kz_lo = max(0, -iz0), kz_hi = min(C.kd, C.din - iz0);
    const int ky_lo = max(0, -iy0), ky_hi = min(C.kh, C.hin - iy0);
    const int kx_lo = max(0, -ix0), kx_hi = min(C.kw, C.win - ix0);
    const int KK = C.kd * C.kh * C.kw;
    const float *tp = STAGED_TAPS ? taps + (size_t)(co - co_base) * C.cin * KK : C.w + (size_t)co * C.cin * KK;
    float p = 0.0f;
    for (int ci = 0; ci < C.cin; ++ci)
        for (int kz = kz_lo; kz < kz_hi; ++kz)
            for (int ky = ky_lo; ky < ky_hi; ++ky) {
                const int row = ((ci * C.din + iz0 + kz) * C.hin + iy0 + ky) * C.win + ix0;   // source bit of tap kx = 0
                const int k0 = ((ci * C.kd + kz) * C.kh + ky) * C.kw;
                for (int kx = kx_lo; kx < kx_hi; kx += 32) {
                    const int cnt = min(32, kx_hi - kx), bit0 = row + kx, w0 = bit0 >> 5, sft = bit0 & 31;
                    const uint32_t lo = STAGED_BITS ? sb[w0] : __ldcg(sb + w0);
                    const uint32_t hi = sft + cnt > 32 ? (STAGED_BITS ? sb[w0 + 1] : __ldcg(sb + w0 + 1)) : 0u;
                    uint32_t bits = __funnelshift_r(lo, hi, sft) & (cnt >= 32 ? 0xffffffffu : ((1u << cnt) - 1u));
                    while (bits) {
                        const int k = k0 + kx + __ffs(bits) - 1;
                        bits &= bits - 1;
                        p = p + (STAGED_TAPS ? tp[k] : __ldcg(tp + k));
                    }
                }
            }
    return p + C.b[co];
}

// Conv1dConnection.compute (topology.py:640-656) for one target neuron j = (co, ox) of one sample: the sum of the taps
// whose (zero-padded) input position spiked, in ascending (ci, kx) order from +0, then the bias.  Each channel's valid
// tap run [kx_lo, kx_hi) looks at consecutive source bits: it is cut out of the bit row 32 bits at a time with a funnel
// shift (any kernel length) and only its set bits are visited.  STAGED_BITS / STAGED_TAPS as for gather_conv3d.
template <bool STAGED_BITS, bool STAGED_TAPS>
__device__ __forceinline__ float gather_conv1d(const snn_conn_t &C, const uint32_t *sb, const float *taps, int co_base, int j, bool valid) {
    if (!valid) return 0.0f;
    const int co = j / C.wout, ox = j - co * C.wout, ix0 = ox * C.sw - C.pw;
    const int kx_lo = max(0, -ix0), kx_hi = min(C.kw, C.win - ix0);
    const float *tp = STAGED_TAPS ? taps + (size_t)(co - co_base) * C.cin * C.kw : C.w + (size_t)co * C.cin * C.kw;
    float p = 0.0f;
    for (int ci = 0; ci < C.cin; ++ci) {
        const int row = ci * C.win + ix0, k0 = ci * C.kw;   // source bit of tap kx = 0, its tap index
        for (int kx = kx_lo; kx < kx_hi; kx += 32) {
            const int cnt = min(32, kx_hi - kx), bit0 = row + kx, w0 = bit0 >> 5, sft = bit0 & 31;
            const uint32_t lo = STAGED_BITS ? sb[w0] : __ldcg(sb + w0);
            const uint32_t hi = sft + cnt > 32 ? (STAGED_BITS ? sb[w0 + 1] : __ldcg(sb + w0 + 1)) : 0u;
            uint32_t bits = __funnelshift_r(lo, hi, sft) & (cnt >= 32 ? 0xffffffffu : ((1u << cnt) - 1u));
            while (bits) {
                const int k = k0 + kx + __ffs(bits) - 1;
                bits &= bits - 1;
                p = p + (STAGED_TAPS ? tp[k] : __ldcg(tp + k));
            }
        }
    }
    return p + C.b[co];
}

// LocalConnection2D.compute (topology.py:1717-1740) for target neuron j = (f, oy, ox) of one sample (n target neurons):
// per input channel the sum of its own weights w[ci, j, k] whose window position k spiked (k ascending, from +0), then
// the channel sums in ascending ci (the reference's sum(-1).sum(1)).  The kw window bits of a kernel row are cut out of
// the bit row 32 at a time, as in gather_conv.  The weights are read where they are: a lane walks its own contiguous row
// w[ci, j, :] (K floats), so the set bits of one row land in the same 32-byte sectors.  A weight under a silent input is
// never read, which differs from the reference's s_unfold * w for a non-finite weight (DESIGN.md section 8).
// D3: LocalConnection3D.compute (topology.py:1866-1896), j = (f, oz, oy, ox), the same sums with the kernel rows
// (ci, kz, ky) of the depth axis (din / kd / sd / dout, snn_b200.h SNN_CONN_LOCAL3D); without it the depth term is 1 and
// the depth fields, which a LocalConnection2D leaves as the sparse storage, are never read.
template <bool STAGED_BITS, bool D3 = false>
__device__ __forceinline__ float gather_local2d(const snn_conn_t &C, const uint32_t *sb, int n, int j, bool valid) {
    if (!valid) return 0.0f;
    const int kd = D3 ? C.kd : 1, din = D3 ? C.din : 1, HW = C.hout * C.wout;
    const int K = kd * C.kh * C.kw, P = (D3 ? C.dout : 1) * HW, l = j % P;
    const int oz = D3 ? l / HW : 0, r = l - oz * HW, oy = r / C.wout, ox = r - oy * C.wout;
    float p = 0.0f;
    for (int ci = 0; ci < C.cin; ++ci) {
        const float *wr = C.w + ((size_t)ci * n + j) * K;
        float q = 0.0f;
        for (int kz = 0; kz < kd; ++kz)
            for (int ky = 0; ky < C.kh; ++ky) {
                const int row = ((ci * din + (D3 ? oz * C.sd + kz : 0)) * C.hin + oy * C.sh + ky) * C.win + ox * C.sw;
                const int krow = (kz * C.kh + ky) * C.kw;
                for (int kx0 = 0; kx0 < C.kw; kx0 += 32) {
                    const int cnt = min(32, C.kw - kx0), bit0 = row + kx0, w0 = bit0 >> 5, sft = bit0 & 31;
                    const uint32_t lo = STAGED_BITS ? sb[w0] : __ldcg(sb + w0);
                    const uint32_t hi = sft + cnt > 32 ? (STAGED_BITS ? sb[w0 + 1] : __ldcg(sb + w0 + 1)) : 0u;
                    uint32_t bits = __funnelshift_r(lo, hi, sft) & (cnt >= 32 ? 0xffffffffu : ((1u << cnt) - 1u));
                    while (bits) {
                        const int k = krow + kx0 + __ffs(bits) - 1;
                        bits &= bits - 1;
                        q = q + __ldcg(wr + k);
                    }
                }
            }
        p = p + q;
    }
    return p;
}

// ---------------------------------------------------------------------------------------
// MaxPool2dConnection (SNN_CONN_MAXPOOL2D, topology.py:1124-1211) and MaxPoo3dConnection (SNN_CONN_MAXPOOL3D,
// :1214-1301).
//
// The rates the gather of step t reads fold in the spikes that gather reads: step t - 1's (slot rd), or step t's in
// one-step mode when the source comes earlier in the insertion order (`cur`).  Whoever finalises source neuron k of a
// sample writes its next rate, one slot ahead of the readers: in step t the rates of step t + 1 (or, `cur`, of step t,
// which its target reads after the layer barrier of one-step mode).  The window prologue writes the rates of step 0
// from the caller's buffer and the incoming spikes.  No grid barrier is added.
__device__ __forceinline__ void pool_rate_step(const DevNet &N, int li, size_t k, int t, bool sf) {
    for (int c = 0; c < N.n_conns; ++c) {
        const snn_conn_t &C = N.conns[c];
        if (!snn_is_maxpool(C.kind) || C.src != li) continue;
        const bool cur = N.one_step && C.src < C.tgt;
        const int tw = cur ? t : t + 1;   // the step whose gather reads what is written here
        if (tw >= N.T) continue;
        const float r = __ldcg(pool_rates_at(N, c, pool_rate_slot(N.T, tw - 1)) + k);
        pool_rates_at(N, c, pool_rate_slot(N.T, tw))[k] = pool_rate_update(r, C.pool_decay, sf);
    }
}

// The source neuron whose spike target neuron j = (ch, oy, ox) of a sample receives (D3: j = (ch, oz, oy, ox)): the first
// maximum of the rates `r` ([C, hin, win] of that sample; D3: [C, din, hin, win]) over the window — row-major window
// order ((kz,) ky, kx), padding never chosen, strict comparison (an equal rate, -0 against +0 included, keeps the earlier
// element), a NaN taking over as it does in F.max_pool2d's / F.max_pool3d's CPU kernel.  Only D3 reads the depth fields
// (on a MaxPool2dConnection they overlay the NULL sparse pointers).  Plan validation (snn_pool_geometry_ok) guarantees a
// valid element in every window.
template <bool D3 = false>
__device__ __forceinline__ int pool_argmax(const snn_conn_t &C, const float *r, int j) {
    const int L = C.hout * C.wout * (D3 ? C.dout : 1), ch = j / L, l = j - ch * L;
    const int oz = D3 ? l / (C.hout * C.wout) : 0, lp = D3 ? l - oz * (C.hout * C.wout) : l, oy = lp / C.wout, ox = lp - oy * C.wout;
    const int HW = C.hin * C.win, V = HW * (D3 ? C.din : 1);
    const float *rc = r + (size_t)ch * V;
    float best = 0.0f;
    int idx = 0;
    bool any = false;
    const int kd = D3 ? C.kd : 1;
    for (int kz = 0; kz < kd; ++kz) {
        const int iz = D3 ? oz * C.sd - C.pd + kz * C.dd : 0;
        if (D3 && (iz < 0 || iz >= C.din)) continue;
        for (int ky = 0; ky < C.kh; ++ky) {
            const int iy = oy * C.sh - C.ph + ky * C.dh;
            if (iy < 0 || iy >= C.hin) continue;
            for (int kx = 0; kx < C.kw; ++kx) {
                const int ix = ox * C.sw - C.pw + kx * C.dw;
                if (ix < 0 || ix >= C.win) continue;
                const float v = __ldcg(rc + (D3 ? iz * HW : 0) + iy * C.win + ix);
                if (!any || v > best || v != v) { best = v; idx = (D3 ? iz * HW : 0) + iy * C.win + ix; any = true; }
            }
        }
    }
    return ch * V + idx;
}

// Final spikes of one neuron of one sample: traces (nodes.py:96-103), clamp / unclamp (network.py:415-429),
// recordings, and (POOL) the next rate of every MaxPool2d / MaxPoo3dConnection leaving the layer.  Returns the spike that is published.
// (POOL) A PassThroughNodes layer has no traces (its forward never reaches Nodes.forward) and a float32 s.
// (PN) `P` holds the neuron's trace decay and scale (snn_b200.h SNN_NODE_PN).
template <bool POOL, bool PN = false>
__device__ __forceinline__ bool finalize_neuron(const DevNet &N, const DevLayer &D, bool s, float xold, size_t k, int b, int j, int t, int wr,
                                                int li, const NeuronPar *P = nullptr) {
    const snn_layer_t &L = D.L;
    const bool pass = POOL && L.kind == SNN_NODE_PASSTHROUGH;
    bool sf = s;
    if (L.traces && !pass) {
        const float x = PN ? trace_step(xold, s, P->trace_decay, P->trace_scale, L.traces_additive)
                           : trace_step(xold, s, L.trace_decay, L.trace_scale, L.traces_additive);
        L.x[k] = x;
        if (D.xpub) D.xpub[((size_t)wr * N.B + b) * L.n + j] = x;
    }
    if (L.clamp && L.clamp[(L.clamp_per_step ? (size_t)t * L.n : 0) + j]) sf = true;
    if (L.unclamp && L.unclamp[(L.unclamp_per_step ? (size_t)t * L.n : 0) + j]) sf = false;
    if (t == N.T - 1) {
        if (pass) ((float *)L.s)[k] = sf ? 1.0f : 0.0f;
        else L.s[k] = sf ? 1 : 0;
    }
    if (L.rec_s) L.rec_s[((size_t)t * N.B + b) * L.n + j] = sf ? 1 : 0;
    if (L.rec_count && sf) L.rec_count[k] += 1;
    if (POOL) pool_rate_step(N, li, k, t, sf);
    return sf;
}

// ---------------------------------------------------------------------------------------
// phase 1.  Work unit = (layer, 32-neuron tile, chunk of N.cs samples): one warp lane per neuron, the CTA's
// warps stride over the chunk's samples.
// PN: some layer carries per-neuron parameters (snn_b200.h SNN_NODE_PN); a lane loads its neuron's once per unit.
template <bool SPARSE, bool FEAT, bool POOL, bool PN = false>
__device__ void phase1(const DevNet &N, int li, int tile, int chunk, int t, const GenSmem &M) {
    const DevLayer &D = N.layers[li];
    const snn_layer_t &L = D.L;
    const int B = N.B, n = L.n, nw = D.nw;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int j = tile * SNN_TILE + lane;
    const bool valid = j < n;
    const int rd = (t + 1) & 1, wr = t & 1;
    const int b0 = chunk * N.cs, b1 = min(B, b0 + N.cs);
    const bool dc = L.kind == SNN_NODE_DC;
    const bool deferred = dc && L.one_spike;  // final spikes known only after the arg-max
    bool nonbin = false;

    // (a MeanFieldConnection source) the final spikes this warp publishes, counted by lane 0 and added to the layer's
    // count of step t once per unit
    int nsp = 0;
    if (D.spc && tile == 0 && chunk == 0 && threadIdx.x == 0) D.spc[(t + 1) % 3] = 0;   // last read in step t - 1
    if (L.kind == SNN_NODE_INPUT) {
        // Input.forward (nodes.py:211-221): s = x.  Four samples per warp are in flight at once.
        for (int bb = b0 + warp; bb < b1; bb += 4 * SNN_GEN_WARPS) {
            float e[4], xo[4];
            #pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int b = bb + q * SNN_GEN_WARPS;
                const bool ok = valid && b < b1;
                e[q] = (ok && L.ext) ? ld_ext(L, ((size_t)t * B + b) * n + j, nonbin) : 0.0f;
                xo[q] = (ok && L.traces) ? L.x[(size_t)b * n + j] : 0.0f;
            }
            #pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int b = bb + q * SNN_GEN_WARPS;
                if (b >= b1) break;
                const size_t k = (size_t)b * n + j;
                const bool s = e[q] != 0.0f;
                bool sf = false;
                if (valid) {
                    if (L.sum_input) L.summed[k] = L.summed[k] + (s ? 1.0f : 0.0f);
                    sf = finalize_neuron<POOL>(N, D, s, xo[q], k, b, j, t, wr, li);
                }
                const uint32_t fw = __ballot_sync(0xffffffffu, valid && sf);
                if (lane == 0) {
                    D.bits[((size_t)wr * B + b) * nw + tile] = fw;
                    if (D.anyf && fw) atomicOr(D.anyf + (size_t)(t % 3) * B + b, 1u);
                    if (D.spc) nsp += __popc(fw);
                }
            }
        }
        if (D.spc && nsp) atomicAdd(D.spc + t % 3, nsp);
        if (D.anyf && tile == 0)
            for (int b = b0 + threadIdx.x; b < b1; b += SNN_GEN_THREADS) D.anyf[(size_t)((t + 1) % 3) * B + b] = 0u;
        if (nonbin && N.err) atomicOr(N.err, SNN_ERR_NONBINARY);
        return;
    }

    // adaptive threshold (nodes.py:1078-1079, 1093-1094).  The batch sum of a step's threshold crossers is an
    // integer accumulated with atomics over the sample chunks (thcnt[t % 3]); every unit rebuilds the value the
    // previous step left — thdec (the decayed threshold that step used) + theta_plus * count — so no unit waits
    // for another one; chunk 0 publishes this step's decayed value and clears the counter slot of step t + 1.
    NeuronPar P;
    if (PN) P = neuron_par(L, valid ? j : 0);
    float theta = 0.0f;
    if (dc && valid) {
        if (L.learning) {
            const float tplus = PN ? P.theta_plus : L.theta_plus;
            const float prev = t == 0 ? L.theta[j]
                                      : __ldcg(D.thdec + (size_t)rd * n + j) + tplus * (float)__ldcg(D.thcnt + (size_t)((t + 2) % 3) * n + j);
            theta = prev * (PN ? P.theta_decay : L.theta_decay);
            if (chunk == 0 && warp == 0) {
                D.thdec[(size_t)wr * n + j] = theta;
                D.thcnt[(size_t)((t + 1) % 3) * n + j] = 0;
            }
        } else {
            theta = L.theta[j];
        }
    }
    int cnt = 0;  // candidates of this column over this warp's samples

    // a convolutional input: stage the chunk's source bit rows and the taps of this tile's output channels (POOL: a
    // Conv3dConnection input likewise, with the depth axis in its channel size and taps; a Conv1dConnection input too,
    // its height axis 1; a LocalConnection2D or LocalConnection3D input gets its bit rows staged the same way, its
    // weights are per target, not taps)
    int conv_c = -1, conv_slot = 0, co_base = 0;
    bool st_bits = false, st_taps = false;
    ConvGeo geo = {};
    for (int c = 0; c < N.n_conns && conv_c < 0; ++c)
        if (N.conns[c].tgt == li &&
            (N.conns[c].kind == SNN_CONN_CONV2D ||
             (POOL && (N.conns[c].kind == SNN_CONN_LOCAL2D || N.conns[c].kind == SNN_CONN_CONV3D || N.conns[c].kind == SNN_CONN_CONV1D ||
                      N.conns[c].kind == SNN_CONN_LOCAL3D))))
            conv_c = c;
    if (conv_c >= 0) {
        const snn_conn_t &C = N.conns[conv_c];
        const DevLayer &S = N.layers[C.src];
        geo = conv_geo(C, j, valid);
        conv_slot = (N.one_step && C.src < li) ? wr : rd;
        const int words = (b1 - b0) * S.nw;
        st_bits = words <= SNN_CONV_STAGE_WORDS;
        const bool c3 = POOL && C.kind == SNN_CONN_CONV3D;
        const int Lhw = C.hout * C.wout * (c3 ? C.dout : 1), K = C.cin * C.kh * C.kw * (c3 ? C.kd : 1);
        co_base = (tile * SNN_TILE) / Lhw;
        const int co_hi = min(n - 1, tile * SNN_TILE + SNN_TILE - 1) / Lhw;
        const int ntaps = (co_hi - co_base + 1) * K;
        st_taps = ntaps <= SNN_CONV_STAGE_TAPS && (!POOL || (C.kind != SNN_CONN_LOCAL2D && C.kind != SNN_CONN_LOCAL3D));
        if (st_bits) {
            const uint32_t *src = S.bits + ((size_t)conv_slot * B + b0) * S.nw;
            for (int k0 = threadIdx.x; k0 < words; k0 += 4 * SNN_GEN_THREADS) {
                uint32_t wq[4];
                #pragma unroll
                for (int q = 0; q < 4; ++q) wq[q] = k0 + q * SNN_GEN_THREADS < words ? __ldcg(src + k0 + q * SNN_GEN_THREADS) : 0u;
                #pragma unroll
                for (int q = 0; q < 4; ++q)
                    if (k0 + q * SNN_GEN_THREADS < words) M.cbits[k0 + q * SNN_GEN_THREADS] = wq[q];
            }
        }
        if (st_taps)
            for (int k = threadIdx.x; k < ntaps; k += SNN_GEN_THREADS) M.xs[k] = __ldcg(C.w + (size_t)co_base * K + k);
        __syncthreads();
    }
    uint16_t *lst = M.list + warp * SNN_GATHER_BLOCK;
    // the incoming connections in insertion order (the first four get their first bit words prefetched)
    int cl[4] = {-1, -1, -1, -1}, ncl = 0, nin = 0;
    for (int c = 0; c < N.n_conns; ++c)
        if (N.conns[c].tgt == li) {
            #pragma unroll
            for (int q = 0; q < 4; ++q)
                if (q == ncl && nin < 4) cl[q] = c;
            if (nin < 4) ++ncl;
            ++nin;
        }

    // first bit words of the dense inputs and the "sample spiked at all" flags of wide sources, fetched one sample
    // ahead: the gather of sample b starts without waiting for L2
    uint32_t fwn[4], afn[4];
    auto prefetch = [&](int b) {
        #pragma unroll
        for (int q = 0; q < 4; ++q) {
            fwn[q] = 0u; afn[q] = 1u;
            if (q < ncl && b < b1 && N.conns[cl[q]].kind != SNN_CONN_CONV2D && N.conns[cl[q]].kind != SNN_CONN_MEANFIELD &&
                !(SPARSE && N.conns[cl[q]].kind == SNN_CONN_SPARSE) && !(POOL && snn_pool_inst_kind(N.conns[cl[q]].kind))) {
                const snn_conn_t &C = N.conns[cl[q]];
                const DevLayer &S = N.layers[C.src];
                const int slot = (N.one_step && C.src < li) ? wr : rd;
                if (lane < S.nw) fwn[q] = __ldcg(S.bits + ((size_t)slot * B + b) * S.nw + lane);
                if (S.anyf) afn[q] = __ldcg(S.anyf + (size_t)(slot == wr ? t % 3 : (t + 2) % 3) * B + b);
            }
        }
    };
    prefetch(b0 + warp);

    for (int b = b0 + warp; b < b1; b += SNN_GEN_WARPS) {
        const size_t k = (size_t)b * n + j;
        uint32_t fw[4], af[4];
        #pragma unroll
        for (int q = 0; q < 4; ++q) { fw[q] = fwn[q]; af[q] = afn[q]; }
        prefetch(b + SNN_GEN_WARPS);
        float v = 0.0f, rc = 0.0f, xold = 0.0f, ic = 0.0f;
        if (valid && !(POOL && L.kind == SNN_NODE_PASSTHROUGH)) {   // (PassThroughNodes: no v, refrac_count, traces)
            v = L.v[k];
            if (L.kind != SNN_NODE_MCP) rc = L.refrac_count[k];
            if (L.traces && !deferred) xold = L.x[k];
            if (L.kind == SNN_NODE_CURRENT_LIF) ic = L.i[k];
        }
        // network.py:211-250: accumulate every incoming connection in insertion order
        float cur = 0.0f;
        const bool has_in = nin > 0;
        int seen = 0;
        for (int c = 0; c < N.n_conns; ++c) {
            const snn_conn_t &C = N.conns[c];
            if (C.tgt != li) continue;
            const DevLayer &S = N.layers[C.src];
            uint32_t first = 0u, anysp = 1u;
            #pragma unroll
            for (int q = 0; q < 4; ++q)
                if (q == seen) { first = fw[q]; anysp = af[q]; }
            const bool prefetched = seen < 4;
            ++seen;
            // one-step mode (network.py:393-396): sources earlier in the insertion order have already
            // produced this step's spikes (slot wr); everything else is still at step t-1 (slot rd)
            const int slot = (N.one_step && C.src < li) ? wr : rd;
            float p;
            if (C.kind == SNN_CONN_CONV2D) {
                const uint32_t *gsb = S.bits + ((size_t)slot * B + b) * S.nw;
                if (c == conv_c && st_bits) {
                    const uint32_t *ssb = M.cbits + (size_t)(b - b0) * S.nw;
                    p = st_taps ? gather_conv<true, true>(C, ssb, M.xs, co_base, j, valid, geo) : gather_conv<true, false>(C, ssb, nullptr, 0, j, valid, geo);
                } else if (c == conv_c && st_taps) {
                    p = gather_conv<false, true>(C, gsb, M.xs, co_base, j, valid, geo);
                } else {
                    p = gather_conv<false, false>(C, gsb, nullptr, 0, j, valid, c == conv_c ? geo : conv_geo(C, j, valid));
                }
            } else if (POOL && snn_is_maxpool(C.kind)) {   // rates of this step: pool_rate_step / the prologue
                const float *r = pool_rates_at(N, c, pool_rate_slot(N.T, t)) + (size_t)b * S.L.n;
                const uint32_t *sb = S.bits + ((size_t)slot * B + b) * S.nw;
                const int i = !valid ? 0 : C.kind == SNN_CONN_MAXPOOL3D ? pool_argmax<true>(C, r, j) : pool_argmax<false>(C, r, j);
                p = (valid && ((__ldcg(sb + (i >> 5)) >> (i & 31)) & 1u)) ? 1.0f : 0.0f;
            } else if (POOL && C.kind == SNN_CONN_CONV3D) {
                const uint32_t *gsb = S.bits + ((size_t)slot * B + b) * S.nw;
                if (c == conv_c && st_bits) {
                    const uint32_t *ssb = M.cbits + (size_t)(b - b0) * S.nw;
                    p = st_taps ? gather_conv3d<true, true>(C, ssb, M.xs, co_base, j, valid) : gather_conv3d<true, false>(C, ssb, nullptr, 0, j, valid);
                } else if (c == conv_c && st_taps) {
                    p = gather_conv3d<false, true>(C, gsb, M.xs, co_base, j, valid);
                } else {
                    p = gather_conv3d<false, false>(C, gsb, nullptr, 0, j, valid);
                }
            } else if (POOL && C.kind == SNN_CONN_CONV1D) {
                const uint32_t *gsb = S.bits + ((size_t)slot * B + b) * S.nw;
                if (c == conv_c && st_bits) {
                    const uint32_t *ssb = M.cbits + (size_t)(b - b0) * S.nw;
                    p = st_taps ? gather_conv1d<true, true>(C, ssb, M.xs, co_base, j, valid) : gather_conv1d<true, false>(C, ssb, nullptr, 0, j, valid);
                } else if (c == conv_c && st_taps) {
                    p = gather_conv1d<false, true>(C, gsb, M.xs, co_base, j, valid);
                } else {
                    p = gather_conv1d<false, false>(C, gsb, nullptr, 0, j, valid);
                }
            } else if (POOL && C.kind == SNN_CONN_LOCAL2D) {
                p = c == conv_c && st_bits ? gather_local2d<true>(C, M.cbits + (size_t)(b - b0) * S.nw, n, j, valid)
                                           : gather_local2d<false>(C, S.bits + ((size_t)slot * B + b) * S.nw, n, j, valid);
            } else if (POOL && C.kind == SNN_CONN_LOCAL3D) {
                p = c == conv_c && st_bits ? gather_local2d<true, true>(C, M.cbits + (size_t)(b - b0) * S.nw, n, j, valid)
                                           : gather_local2d<false, true>(C, S.bits + ((size_t)slot * B + b) * S.nw, n, j, valid);
            } else if (C.kind == SNN_CONN_MEANFIELD) {   // s.float().mean() * w (snn_b200.h): the source's count of the step
                const int cnt_s = __ldcg(S.spc + (slot == wr ? t % 3 : (t + 2) % 3));
                const float mean = (float)cnt_s / (float)(B * S.L.n);
                p = valid ? mean * C.w[C.mf_off[j] + (size_t)b * C.mf_stride] : 0.0f;
            } else if (SPARSE && C.kind == SNN_CONN_SPARSE) {   // gathered by phase_sparse ahead of this phase
                p = valid ? __ldcg(N.sp[c].out + (size_t)b * n + j) : 0.0f;
                if (C.b && valid) p = p + C.b[j];
            } else {
                const uint32_t *sbr = S.bits + ((size_t)slot * B + b) * S.nw;
                if (!prefetched) first = lane < S.nw ? __ldcg(sbr + lane) : 0u;
                p = anysp ? gather<FEAT>(C, sbr, S.nw, S.L.n, n, j, valid, lane, lst, first, N.seed, (uint32_t)t + N.step_offset, (uint32_t)c)
                          : 0.0f;
                if (C.b && valid) p = p + C.b[j];
            }
            cur = cur + p;
        }
        bool s = false;
        if (valid) {
            // (one-step mode: the connection input REPLACES the external one, network.py:393-396)
            if (L.ext && !(N.one_step && has_in)) { bool nb = false; cur = cur + ld_ext(L, ((size_t)t * B + b) * n + j, nb); }
            if (L.inject_v) v = v + L.inject_v[(L.inject_per_step ? (size_t)t * n : 0) + j];  // network.py:398-404
            float xin = cur;
            const bool pass = POOL && L.kind == SNN_NODE_PASSTHROUGH;   // no v, refrac_count or summed of its own
            if (pass) {   // PassThroughNodes.forward (conversion/nodes.py:137-144): s = x
                s = xin != 0.0f;
                nonbin |= s && xin != 1.0f;
            } else if (dc) {
                s = PN ? dc_step_p(L, P.decay, P.rest, P.thresh, v, rc, xin, theta) : dc_step(L, v, rc, xin, theta);
                if (L.has_lbound && v < L.lbound) v = L.lbound;  // nodes.py:1108-1109
            } else if (L.kind == SNN_NODE_IF) {
                s = if_step(L, v, rc, xin);
            } else if (L.kind == SNN_NODE_CURRENT_LIF) {
                s = clif_step(L, v, rc, ic, xin);
                L.i[k] = ic;
            } else if (L.kind == SNN_NODE_BOOSTED_LIF) {
                s = boosted_step(L, v, rc, xin);
            } else if (L.kind == SNN_NODE_MCP) {   // McCullochPitts.forward (nodes.py:278-288): voltages equal the inputs
                v = xin;
                s = v >= L.thresh;
            } else if (POOL && L.kind == SNN_NODE_SUBIF) {
                s = subif_step(L, v, rc, xin);
            } else {
                s = PN ? lif_step_p(L, P.decay, P.rest, P.thresh, v, rc, xin) : lif_step(L, v, rc, xin);
            }
            if (!pass) {
                L.v[k] = v;
                if (L.kind != SNN_NODE_MCP) L.refrac_count[k] = rc;
                if (L.sum_input) L.summed[k] = L.summed[k] + xin;
                if (L.rec_v) L.rec_v[((size_t)t * B + b) * n + j] = v;
            }
            cnt += s ? 1 : 0;
        }
        const uint32_t word = __ballot_sync(0xffffffffu, valid && s);
        if (deferred) {
            if (lane == 0) D.candbits[(size_t)b * nw + tile] = word;
            if (word) {
                unsigned long long key = 0ull;
                if (valid && s) key = snn_one_spike_key(N.seed, (uint32_t)t + N.step_offset, (uint32_t)li, (uint32_t)b, (uint32_t)j);
                #pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
                    const unsigned long long other = __shfl_xor_sync(0xffffffffu, key, o);
                    key = other > key ? other : key;
                }
                if (lane == 0) atomicMax(D.keys + (size_t)wr * B + b, key);
            }
        } else {
            bool sf = false;
            if (valid) sf = finalize_neuron<POOL, PN>(N, D, s, xold, k, b, j, t, wr, li, &P);
            const uint32_t fw = __ballot_sync(0xffffffffu, valid && sf);
            if (lane == 0) {
                D.bits[((size_t)wr * B + b) * nw + tile] = fw;
                if (D.anyf && fw) atomicOr(D.anyf + (size_t)(t % 3) * B + b, 1u);
                if (D.spc) nsp += __popc(fw);
            }
        }
    }
    if (D.spc && nsp) atomicAdd(D.spc + t % 3, nsp);
    if (D.anyf && tile == 0)   // the flag slot of step t + 1 (last read in step t - 1)
        for (int b = b0 + threadIdx.x; b < b1; b += SNN_GEN_THREADS) D.anyf[(size_t)((t + 1) % 3) * B + b] = 0u;

    if (POOL && nonbin && N.err) atomicOr(N.err, SNN_ERR_NONBINARY);   // a PassThroughNodes input outside {0, 1}
    // theta += theta_plus * sum_b s  (nodes.py:1093-1094)
    if (dc && L.learning && valid && cnt > 0) atomicAdd(D.thcnt + (size_t)(t % 3) * n + j, cnt);
    if (deferred && tile == 0) {
        // clear the key slot the NEXT step will arg-max into (last read two barriers ago)
        for (int b = b0 + threadIdx.x; b < b1; b += SNN_GEN_THREADS) D.keys[(size_t)rd * B + b] = 0ull;
    }
    if (conv_c >= 0) __syncthreads();   // the staged rows / taps are overwritten by the CTA's next unit
}

// ---------------------------------------------------------------------------------------
// phase 2 (DiehlAndCookNodes with one_spike): keep the arg-max candidate of each sample
// (nodes.py:1097-1105), then traces / clamp / publish as in phase 1.  Same work units as phase 1.  PN: as for phase 1.
template <bool POOL, bool PN = false>
__device__ void phase2(const DevNet &N, int li, int tile, int chunk, int t) {
    const DevLayer &D = N.layers[li];
    const snn_layer_t &L = D.L;
    const int B = N.B, n = L.n, nw = D.nw;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int j = tile * SNN_TILE + lane;
    const bool valid = j < n;
    NeuronPar P;
    if (PN) P = neuron_par(L, valid ? j : 0);
    const int wr = t & 1;
    const int b0 = chunk * N.cs, b1 = min(B, b0 + N.cs);
    int nsp = 0;   // (a MeanFieldConnection source) the winners this warp publishes, as in phase 1
    for (int bb = b0 + warp; bb < b1; bb += 4 * SNN_GEN_WARPS) {
        uint32_t cand[4];
        unsigned long long key[4];
        float xo[4];
        #pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int b = bb + q * SNN_GEN_WARPS;
            const bool ok = b < b1;
            cand[q] = ok ? __ldcg(D.candbits + (size_t)b * nw + tile) : 0u;
            key[q] = ok ? __ldcg(D.keys + (size_t)wr * B + b) : 0ull;
            xo[q] = (ok && valid && L.traces) ? L.x[(size_t)b * n + j] : 0.0f;
        }
        #pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int b = bb + q * SNN_GEN_WARPS;
            if (b >= b1) break;
            const size_t k = (size_t)b * n + j;
            const bool s = valid && ((cand[q] >> lane) & 1u) && key[q] != 0ull && (uint32_t)(key[q] & 0xffffffffull) == (uint32_t)j;
            bool sf = false;
            if (valid) sf = finalize_neuron<POOL, PN>(N, D, s, xo[q], k, b, j, t, wr, li, &P);
            const uint32_t fw = __ballot_sync(0xffffffffu, valid && sf);
            if (lane == 0) {
                D.bits[((size_t)wr * B + b) * nw + tile] = fw;
                if (D.anyf && fw) atomicOr(D.anyf + (size_t)(t % 3) * B + b, 1u);
                if (D.spc) nsp += __popc(fw);
            }
        }
    }
    if (D.spc && nsp) atomicAdd(D.spc + t % 3, nsp);
}

// ---------------------------------------------------------------------------------------
// phase 3: learning-rule update of the rows [wg0*32, wg1*32) of one weight tile W[:, tile] of connection `ci`.
//   U[i,j] = reduce_b s_src[b,i] * (x_tgt[b,j] * nu0)      pre-synaptic term
//   V[i,j] = reduce_b x_src[b,i] * (s_tgt[b,j] * nu1)      post-synaptic term
// Both reduce over the batch in ascending b.  The reference materialises [B,n_src,n_tgt]
// (learning.py:399-417, MCC_learning.py:234-299); here only rows with a pre-synaptic spike
// and columns with a post-synaptic spike are touched (everything else is a bitwise no-op),
// except when a full pass is required: weight decay != 1, or the first update of the window
// (entries may sit outside [wmin, wmax] after normalize()).
// Work unit = (connection, tile, row chunk): the target traces of the tile are staged in shared memory once
// (every row group reads them), a warp owns one group of 32 source rows at a time, stages the pre-synaptic
// traces of the (few) samples with a post-synaptic event for those rows, and rewrites the rows eight at a time
// so that eight weight loads are in flight.
// SYN: the connection may carry per-synapse bounds and rates (snn_b200.h wmin_t ...); plans without them run the
// instantiation that never reads those fields.
template <bool SYN, bool WN = false>
__device__ void phase3(const DevNet &N, int ci, int tile, int wg0, int wg1, int t, const GenSmem &M) {
    const snn_conn_t &C = N.conns[ci];
    const DevLayer &S = N.layers[C.src], &G = N.layers[C.tgt];
    const int B = N.B, ns = S.L.n, nt = G.L.n, nwS = S.nw, nwG = G.nw;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int j = tile * SNN_TILE + lane;
    const bool valid = j < nt;
    const int wr = t & 1;
    const int NG = (B + 31) / 32;
    const bool stdp = SNN_RULE_IS_STDP(C.rule);
    const bool wdep = C.rule == SNN_RULE_WDEP_POSTPRE || C.rule == SNN_RULE_HEBBIAN;   // plain sums: nu applied after the reduction
    const bool pre_on = stdp && C.nu0 != 0.0f, post_on = stdp && C.nu1 != 0.0f;
    const bool decay_on = C.weight_decay != 0.0f && C.weight_decay != 1.0f;
    // (WN: a connection normalised every step may leave [wmin, wmax] in any row before its update)
    const bool full = decay_on || (C.has_clamp && (t == 0 || (WN && C.norm_step)));
    const float Bf = (float)B;
    const bool stage = pre_on && M.xt != nullptr;
    // PostPre's pre-synaptic rate of my column (per target only, snn_b200.h)
    const float nu0j = SYN ? syn_at(C.nu0_t, C.nu0_form, C.nu0, 0, valid ? j : 0, nt) : C.nu0;

    // Samples whose target-trace row is all zero in this tile cannot change the pre-synaptic term (adding +-0 to a sum
    // that started at +0 is a bitwise no-op), and in networks of rarely spiking neurons that is most of them: the
    // staging pass records the others in `live`, the accumulation looks at nobody else.
    if (stage) {
        if (threadIdx.x < NG) M.live[threadIdx.x] = 0u;
        __syncthreads();
        for (int b0 = warp; b0 < B; b0 += 8 * SNN_GEN_WARPS) {   // eight rows of the trace tile in flight per warp
            float tx[8];
            #pragma unroll
            for (int q = 0; q < 8; ++q) {
                const int b = b0 + q * SNN_GEN_WARPS;
                tx[q] = (valid && b < B) ? __ldcg(G.L.x + (size_t)b * nt + j) : 0.0f;
            }
            #pragma unroll
            for (int q = 0; q < 8; ++q) {
                const int b = b0 + q * SNN_GEN_WARPS;
                if (b < B) {
                    const float v = wdep ? tx[q] : tx[q] * nu0j;
                    M.xt[b * 32 + lane] = v;
                    const bool nzrow = __any_sync(0xffffffffu, v != 0.0f);
                    if (lane == 0 && nzrow) atomicOr(M.live + (b >> 5), 1u << (b & 31));
                }
            }
        }
    }

    // column events: colmask[g*32 + lane] = samples of group g whose target spike hit column j
    uint32_t colany = 0;
    if (post_on) {
        for (int b = threadIdx.x; b < B; b += SNN_GEN_THREADS) M.evslot[b] = 0xFF;
        for (int g = warp; g < NG; g += SNN_GEN_WARPS) {
            const int b = g * 32 + lane;
            const uint32_t wb = b < B ? __ldcg(G.bits + ((size_t)wr * B + b) * nwG + tile) : 0u;
            uint32_t mine = 0;
            if (__any_sync(0xffffffffu, wb != 0u)) {
                #pragma unroll
                for (int r = 0; r < 32; ++r) {
                    const uint32_t m = __ballot_sync(0xffffffffu, (wb >> r) & 1u);
                    if (lane == r) mine = m;
                }
            }
            M.colmask[g * 32 + lane] = mine;
        }
        __syncthreads();
        for (int g = 0; g < NG; ++g) colany |= M.colmask[g * 32 + lane];
        // the first SNN_P3_MAXEV samples (ascending) with an event in this tile get a staging slot
        if (warp == 0) {
            int nev = 0;
            for (int g = 0; g < NG; ++g) {
                uint32_t m = M.colmask[g * 32 + lane];
                #pragma unroll
                for (int o = 16; o > 0; o >>= 1) m |= __shfl_xor_sync(0xffffffffu, m, o);
                if (lane == 0)
                    while (m && nev < SNN_P3_MAXEV) {
                        const int bb = g * 32 + __ffs(m) - 1;
                        m &= m - 1;
                        M.evb[nev] = bb;
                        M.evslot[bb] = (uint8_t)nev;
                        ++nev;
                    }
            }
            if (lane == 0) M.evb[SNN_P3_MAXEV] = nev;
        }
    }
    const bool any_col = __syncthreads_or(colany != 0u) != 0;   // also publishes xt / evb / evslot
    if (!full && !pre_on && !any_col) return;

    float *acc = M.acc + warp * (32 * 32);
    for (int r = 0; r < 32; ++r) acc[r * 32 + lane] = 0.0f;
    float *xsw = M.xs + warp * (SNN_P3_MAXEV * 32);
    const int nev = any_col ? M.evb[SNN_P3_MAXEV] : 0;
    __syncwarp();

    // In the dense regime (large batches: nearly every source row has a spike somewhere in the batch) the weight rows
    // of a group are fetched before it is known which of them change — their L2 round trip then hides behind the
    // accumulation; for small batches only the rows that need it are read.
    const bool eager = B >= 64;
    const bool post_t = colany != 0u;
    for (int wg = wg0 + warp; wg < wg1; wg += SNN_GEN_WARPS) {
        const int i0 = wg * 32;
        float wv[8];
        if (eager) {
            #pragma unroll
            for (int q = 0; q < 8; ++q) wv[q] = (valid && i0 + q < ns) ? __ldcg(C.w + (size_t)(i0 + q) * nt + j) : 0.0f;
        }
        if (nev > 0) {   // pre-synaptic traces of the event samples for my 32 rows (coalesced, four in flight)
            const int i = i0 + lane;
            for (int e0 = 0; e0 < nev; e0 += 4) {
                float xv[4];
                #pragma unroll
                for (int q = 0; q < 4; ++q)
                    xv[q] = (e0 + q < nev && i < ns) ? __ldcg(S.xpub + ((size_t)wr * B + M.evb[min(e0 + q, nev - 1)]) * ns + i) : 0.0f;
                #pragma unroll
                for (int q = 0; q < 4; ++q)
                    if (e0 + q < nev) xsw[(e0 + q) * 32 + lane] = xv[q];
            }
        }
        uint32_t tmask = 0, umask = 0;   // rows with a pre-synaptic spike / with a non-zero contribution to U
        if (pre_on) {
            for (int g0 = 0; g0 < NG; g0 += 8) {
                uint32_t mine[8];
                #pragma unroll
                for (int q = 0; q < 8; ++q) {
                    const int bl = (g0 + q) * 32 + lane;
                    mine[q] = (g0 + q < NG && bl < B) ? __ldcg(S.bits + ((size_t)wr * B + bl) * nwS + wg) : 0u;
                }
                #pragma unroll
                for (int q = 0; q < 8; ++q) {
                    uint32_t nz = __ballot_sync(0xffffffffu, mine[q] != 0u);
                    {   // every spiking sample marks its rows; only the live ones are accumulated
                        uint32_t orw = mine[q];
                        #pragma unroll
                        for (int o = 16; o > 0; o >>= 1) orw |= __shfl_xor_sync(0xffffffffu, orw, o);
                        tmask |= orw;
                    }
                    if (stage && g0 + q < NG) nz &= M.live[g0 + q];
                    while (nz) {
                        const int bb = __ffs(nz) - 1;
                        nz &= nz - 1;
                        uint32_t word = __shfl_sync(0xffffffffu, mine[q], bb);
                        const int b = (g0 + q) * 32 + bb;
                        float tx = 0.0f;
                        if (stage) {
                            tx = M.xt[b * 32 + lane];
                        } else {
                            if (valid) {
                                tx = __ldcg(G.L.x + (size_t)b * nt + j);
                                if (!wdep) tx = tx * nu0j;
                            }
                            if (!__any_sync(0xffffffffu, tx != 0.0f)) continue;
                        }
                        umask |= word;
                        while (word) {
                            const int r = __ffs(word) - 1;
                            word &= word - 1;
                            acc[r * 32 + lane] = acc[r * 32 + lane] + tx;
                        }
                    }
                }
            }
        }
        __syncwarp();
        if (!full && !(wdep ? tmask : umask) && !any_col) continue;
        // Columns with a post-synaptic event change in every row.  They are few (one spiking neuron in the tile is
        // the rule), so each is rewritten with one lane per ROW — one pass of the rule for all 32 rows of the group —
        // instead of dragging the whole warp through 32 row iterations for the sake of one lane.
        const uint32_t evcols = __ballot_sync(0xffffffffu, post_t);
        for (uint32_t ec = evcols; ec; ec &= ec - 1) {
            const int jl = __ffs(ec) - 1, jc = tile * SNN_TILE + jl, i = i0 + lane;
            if (i < ns) {
                const bool pre_t = (tmask >> lane) & 1u;
                float U = 0.0f, V = 0.0f;
                if (pre_t) {
                    U = acc[lane * 32 + jl];
                    if (C.reduction == SNN_REDUCE_MEAN) U = U / Bf;
                }
                const float nu1c = SYN ? syn_at(C.nu1_t, C.nu1_form, C.nu1, 0, jc, nt) : C.nu1;
                for (int g = 0; g < NG; ++g) {
                    uint32_t m = M.colmask[g * 32 + jl];
                    while (m) {
                        const int b = g * 32 + __ffs(m) - 1;
                        m &= m - 1;
                        const int slot = M.evslot[b];
                        const float xs = slot != 0xFF ? xsw[slot * 32 + lane] : __ldcg(S.xpub + ((size_t)wr * B + b) * ns + i);
                        V = V + xs * (wdep ? 1.0f : nu1c);
                    }
                }
                if (C.reduction == SNN_REDUCE_MEAN) V = V / Bf;
                float *wp = C.w + (size_t)i * nt + jc;
                *wp = SYN ? apply_rule_syn(C, __ldcg(wp), U, pre_t, V, true, i, jc, nt) : apply_rule(C, __ldcg(wp), U, pre_t, V, true);
            }
        }
        __syncwarp();
        for (int r0 = 0; r0 < 32; r0 += 8) {
            bool nd[8];
            bool anyneed = false;
            #pragma unroll
            for (int q = 0; q < 8; ++q) {
                const int r = r0 + q, i = i0 + r;
                const bool pre_t = (tmask >> r) & 1u;
                // a row whose U is +0 in every column is left alone: w - 0 is w, and w has been inside [wmin, wmax] since
                // the full pass of step 0 (the weight-dependent and Hebbian forms compute w + (+-0), which may flip
                // the sign of a zero: they always rewrite)
                const bool touched = wdep ? pre_t : ((umask >> r) & 1u) != 0u;
                nd[q] = valid && i < ns && !post_t && (full || touched);   // event columns: done above
                if (!eager) wv[q] = nd[q] ? __ldcg(C.w + (size_t)i * nt + j) : 0.0f;
                anyneed |= nd[q];
            }
            float wn[8];   // next group's rows: in flight while this group is rewritten
            if (eager && r0 + 8 < 32) {
                #pragma unroll
                for (int q = 0; q < 8; ++q) wn[q] = (valid && i0 + r0 + 8 + q < ns) ? __ldcg(C.w + (size_t)(i0 + r0 + 8 + q) * nt + j) : 0.0f;
            }
            if (__any_sync(0xffffffffu, anyneed)) {
                #pragma unroll
                for (int q = 0; q < 8; ++q) {
                    const int r = r0 + q, i = i0 + r;
                    const bool pre_t = (tmask >> r) & 1u;
                    if (nd[q]) {
                        float U = 0.0f;
                        if (pre_t) {
                            U = acc[r * 32 + lane];
                            if (C.reduction == SNN_REDUCE_MEAN) U = U / Bf;
                        }
                        C.w[(size_t)i * nt + j] = SYN ? apply_rule_syn(C, wv[q], U, pre_t, 0.0f, false, i, j, nt)
                                                      : apply_rule(C, wv[q], U, pre_t, 0.0f, false);
                    }
                }
            }
            #pragma unroll
            for (int q = 0; q < 8; ++q)
                if ((umask >> (r0 + q)) & 1u) acc[(r0 + q) * 32 + lane] = 0.0f;
            if (eager) {
                #pragma unroll
                for (int q = 0; q < 8; ++q) wv[q] = wn[q];
            }
        }
        __syncwarp();
    }
    __syncthreads();
}

// ---------------------------------------------------------------------------------------
// phase 3 for MCC_learning.PostPre with average_update (MCC_learning.py:210-302; snn_b200.h SNN_RULE_AVG).  Same units
// as phase3 (connection, 32-column tile, chunk of source row groups), a warp per row group, a lane per column.  A pre
// slot is zero outside the rows that had a spike in its step and a post slot outside the columns, so the slot bitmaps
// bound every pass: a slot write touches the rows (columns) active now and those of the slot's previous occupant (set to
// zero); the mean of an element sums, in ascending slot order from +0, only the slots whose bitmap covers it (the others
// hold zeros, which leave such a sum as it is); an element no slot covers is left alone.  With large batches nearly
// every row is active and the passes are dense.  Order per element: pre slot, pre mean, post slot, post mean, decay,
// clamp.  The shared accumulators of a warp hold first U (the step's pre-synaptic term), then the pre sums, then V,
// then the post sums.
__device__ void phase3_mcc_avg(const DevNet &N, int ci, int tile, int wg0, int wg1, int t, const GenSmem &M) {
    const snn_conn_t &C = N.conns[ci];
    const DevAvg &A = N.avg[ci];
    const DevLayer &S = N.layers[C.src], &G = N.layers[C.tgt];
    const int B = N.B, ns = S.L.n, nt = G.L.n, nwS = S.nw, nwG = G.nw, K = C.avg_k;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int j = tile * SNN_TILE + lane;
    const bool valid = j < nt;
    const int wr = t & 1, in = (t + N.T) & 1, out = in ^ 1;
    const bool pre_on = C.nu0 != 0.0f, post_on = C.nu1 != 0.0f;
    const bool decay_on = C.weight_decay != 0.0f && C.weight_decay != 1.0f;
    const bool full = decay_on || (C.has_clamp && t == 0);
    const bool mean = C.reduction == SNN_REDUCE_MEAN;
    const float Bf = (float)B, Kf = (float)K;
    const int pp = (C.avg_idx_pre + t) % K, pq = (C.avg_idx_post + t) % K;   // the slots this step writes
    const bool apply_pre = pre_on && (C.avg_continues || (pp + 1) % K == 0);
    const bool apply_post = post_on && (C.avg_continues || (pq + 1) % K == 0);
    const size_t KS = (size_t)ns * nt;
    const uint32_t *rows_in = A.rows[in], *cols_in = A.cols[in];

    // the columns of this tile with a post-synaptic spike now, and those any post slot covers after this step
    // the target traces of the tile times nu0, [B][32], when they fit (read by every row group)
    if (pre_on && M.xt) {
        for (int b = warp; b < B; b += SNN_GEN_WARPS) M.xt[b * 32 + lane] = valid ? __ldcg(G.L.x + (size_t)b * nt + j) * C.nu0 : 0.0f;
        __syncthreads();
    }
    uint32_t cnow = 0, cunion = 0, cold = 0;
    if (post_on) {
        for (int b = lane; b < B; b += 32) cnow |= __ldcg(G.bits + ((size_t)wr * B + b) * nwG + tile);
        #pragma unroll
        for (int o = 16; o > 0; o >>= 1) cnow |= __shfl_xor_sync(0xffffffffu, cnow, o);
        for (int q = 0; q < K; ++q) {
            const uint32_t c = q == pq ? cnow : __ldcg(cols_in + (size_t)q * nwG + tile);
            cunion |= c;
            if (wg0 == 0 && warp == 0 && lane == 0) A.cols[out][(size_t)q * nwG + tile] = c;
        }
        cold = __ldcg(cols_in + (size_t)pq * nwG + tile);
    }
    float *acc = M.acc + warp * (32 * 32);
    for (int wg = wg0 + warp; wg < wg1; wg += SNN_GEN_WARPS) {
        const int i0 = wg * 32;
        const int nr = min(32, ns - i0);
        uint32_t pre_applied = 0;
        if (pre_on) {
            // U of the rows active now: the samples ascending from +0
            for (int r = 0; r < 32; ++r) acc[r * 32 + lane] = 0.0f;
            __syncwarp();
            uint32_t rnow = 0;
            for (int b0 = 0; b0 < B; b0 += 32) {   // a lane per sample fetches the words, the warp walks the non-zero ones
                const uint32_t mw = b0 + lane < B ? __ldcg(S.bits + ((size_t)wr * B + b0 + lane) * nwS + wg) : 0u;
                for (uint32_t nz = __ballot_sync(0xffffffffu, mw != 0u); nz; nz &= nz - 1) {
                    const int b = b0 + __ffs(nz) - 1;
                    uint32_t word = __shfl_sync(0xffffffffu, mw, __ffs(nz) - 1);
                    rnow |= word;
                    const float tx = M.xt ? M.xt[b * 32 + lane] : (valid ? __ldcg(G.L.x + (size_t)b * nt + j) * C.nu0 : 0.0f);
                    while (word) {
                        const int r = __ffs(word) - 1;
                        word &= word - 1;
                        acc[r * 32 + lane] = acc[r * 32 + lane] + tx;
                    }
                }
            }
            const uint32_t rold = __ldcg(rows_in + (size_t)pp * nwS + wg);
            float *slot = C.avg_pre + (size_t)pp * KS;
            for (uint32_t m = rnow | rold; m; m &= m - 1) {
                const int r = __ffs(m) - 1;
                float u = 0.0f;
                if ((rnow >> r) & 1u) {
                    u = acc[r * 32 + lane];
                    if (mean) u = u / Bf;
                }
                if (valid) slot[(size_t)(i0 + r) * nt + j] = u;
            }
            uint32_t runion = 0;
            for (int q = 0; q < K; ++q) {
                const uint32_t rq = q == pp ? rnow : __ldcg(rows_in + (size_t)q * nwS + wg);
                runion |= rq;
                if (tile == 0 && lane == 0) A.rows[out][(size_t)q * nwS + wg] = rq;
            }
            if (apply_pre && runion) {
                __syncwarp();
                for (uint32_t m = runion; m; m &= m - 1) acc[(__ffs(m) - 1) * 32 + lane] = 0.0f;
                for (int q = 0; q < K; ++q) {
                    const uint32_t rq = q == pp ? rnow : __ldcg(rows_in + (size_t)q * nwS + wg);
                    const float *sq = C.avg_pre + (size_t)q * KS + (size_t)i0 * nt + j;
                    for (uint32_t m = rq; m; m &= m - 1) {
                        const int r = __ffs(m) - 1;
                        if (valid) acc[r * 32 + lane] = acc[r * 32 + lane] + __ldcg(sq + (size_t)r * nt);
                    }
                }
                for (uint32_t m = runion; m; m &= m - 1) {
                    const int r = __ffs(m) - 1;
                    float d = acc[r * 32 + lane] / Kf;
                    d = d * C.dt_scale;
                    float *wp = C.w + (size_t)(i0 + r) * nt + j;
                    if (valid) *wp = __ldcg(wp) - d;
                }
                pre_applied = runion;
            }
            __syncwarp();
        }
        const bool col_applied = apply_post && ((cunion >> lane) & 1u);
        if (post_on && (cnow | cold)) {
            // V of the columns active now: the samples ascending from +0, a lane per column, the row's trace broadcast
            for (int r = 0; r < 32; ++r) acc[r * 32 + lane] = 0.0f;
            __syncwarp();
            for (int b0 = 0; b0 < B; b0 += 32) {
                const uint32_t mw = b0 + lane < B ? __ldcg(G.bits + ((size_t)wr * B + b0 + lane) * nwG + tile) : 0u;
                for (uint32_t nz = __ballot_sync(0xffffffffu, mw != 0u); nz; nz &= nz - 1) {
                    const int b = b0 + __ffs(nz) - 1;
                    const uint32_t cw = __shfl_sync(0xffffffffu, mw, __ffs(nz) - 1);
                    const float xs = lane < nr ? __ldcg(S.xpub + ((size_t)wr * B + b) * ns + i0 + lane) : 0.0f;
                    const bool mine = (cw >> lane) & 1u;
                    for (int r = 0; r < nr; ++r) {
                        const float xr = __shfl_sync(0xffffffffu, xs, r);
                        if (mine) acc[r * 32 + lane] = acc[r * 32 + lane] + xr * C.nu1;
                    }
                }
            }
            if (valid && (((cnow | cold) >> lane) & 1u)) {
                float *slot = C.avg_post + (size_t)pq * KS + (size_t)i0 * nt + j;
                const bool now = (cnow >> lane) & 1u;
                for (int r = 0; r < nr; ++r) {
                    float v = 0.0f;
                    if (now) {
                        v = acc[r * 32 + lane];
                        if (mean) v = v / Bf;
                    }
                    slot[(size_t)r * nt] = v;
                }
            }
            __syncwarp();
        }
        if (col_applied) {
            for (int r = 0; r < 32; ++r) acc[r * 32 + lane] = 0.0f;
            for (int q = 0; q < K; ++q) {
                const uint32_t cq = q == pq ? cnow : __ldcg(cols_in + (size_t)q * nwG + tile);
                if (!((cq >> lane) & 1u)) continue;
                const float *sq = C.avg_post + (size_t)q * KS + (size_t)i0 * nt + j;
                for (int r = 0; r < nr; ++r) acc[r * 32 + lane] = acc[r * 32 + lane] + __ldcg(sq + (size_t)r * nt);
            }
        }
        // post mean, decay and clamp of every element a term reached (all of them in a full pass)
        if (valid && (full || col_applied || pre_applied))
            for (int r = 0; r < nr; ++r) {
                if (!(full || col_applied || ((pre_applied >> r) & 1u))) continue;
                float *wp = C.w + (size_t)(i0 + r) * nt + j;
                float w = __ldcg(wp);
                if (col_applied) {
                    float d = acc[r * 32 + lane] / Kf;
                    d = d * C.dt_scale;
                    w = w + d;
                }
                if (C.weight_decay != 0.0f) w = w * C.weight_decay;
                if (C.has_clamp) w = clampf(w, C.wmin, C.wmax);
                *wp = w;
            }
        __syncwarp();
    }
    __syncthreads();   // the staged traces belong to the CTA's next unit
}

// ---------------------------------------------------------------------------------------
// phase 3 for reward-modulated STDP and for convolutional connections.  The rule's state is double
// buffered (DevMstdp): everything is READ from slot `in` and WRITTEN to slot `out`, so no thread
// overwrites a value another thread still needs in this step.
__device__ __forceinline__ float mst_trace(float p, float decay, float a, bool s) {
    // learning.py:1564-1567 / 1999-2003:  P *= exp(-dt/tc);  P += a * s
    const float x = p * decay;
    return x + a * (s ? 1.0f : 0.0f);
}
__device__ __forceinline__ bool bit_of(const uint32_t *row, int i) { return (__ldcg(row + (i >> 5)) >> (i & 31)) & 1u; }

// learning.MSTDP._connection_update (learning.py:1504-1574) + base class decay / clamp (:87-104).
// Work is spread over the tiles of the SOURCE layer (a dense layer's target is often tiny — 10 output
// neurons in BASELINE config 4 — while its source has thousands of rows): unit = 32 rows i (one per
// lane) x all columns j (warps stride over them); the batch sum runs in ascending b per (i, j).  When it
// fits, the rule state the batch loop reads (p_plus and the pre-synaptic spikes of the unit's rows, p_minus
// and the post-synaptic spikes of all columns) is staged in shared memory first, so that the B-long
// dependent loop never waits for L2.  SYN: as for phase3.
template <bool SYN>
__device__ void phase3_mstdp_dense(const DevNet &N, int ci_, int tile, int t, const GenSmem &GS) {
    const snn_conn_t &C = N.conns[ci_];
    const DevMstdp &M = N.mst[ci_];
    const DevLayer &S = N.layers[C.src], &G = N.layers[C.tgt];
    const int B = N.B, ns = S.L.n, nt = G.L.n;
    const int in = (t + N.T) & 1, out = in ^ 1, wr = t & 1;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int i = tile * SNN_TILE + lane;
    const float Bf = (float)B;
    const float *pp = M.pp[in], *pm = M.pm[in];
    const uint8_t *sp = M.sp[in], *st = M.st[in];
    const bool staged = GS.xt != nullptr && (size_t)B * 32 + (size_t)B * nt * 5 + 16 <= sizeof(float) * SNN_GEN_WARPS * 32 * 32;
    float *pp_s = GS.xt;                                   // [B][32]
    float *pm_s = GS.acc;                                  // [B][nt]
    uint8_t *st_s = (uint8_t *)(pm_s + (size_t)B * nt);    // [B][nt]
    uint8_t *sp_s = st_s + ((size_t)B * nt + 15) / 16 * 16;  // [B][32]
    uint32_t *sbw = GS.colmask;                            // [B] source spike word of this tile, step t
    if (staged) {
        for (int b0 = warp; b0 < B; b0 += 8 * SNN_GEN_WARPS) {   // eight samples' rows in flight per warp
            float pv[8]; uint8_t sv[8];
            #pragma unroll
            for (int q = 0; q < 8; ++q) {
                const int b = b0 + q * SNN_GEN_WARPS;
                const bool ok = i < ns && b < B;
                pv[q] = ok ? __ldcg(pp + (size_t)b * ns + i) : 0.0f;
                sv[q] = ok ? __ldcg(sp + (size_t)b * ns + i) : (uint8_t)0;
            }
            #pragma unroll
            for (int q = 0; q < 8; ++q) {
                const int b = b0 + q * SNN_GEN_WARPS;
                if (b < B) { pp_s[b * 32 + lane] = pv[q]; sp_s[b * 32 + lane] = sv[q]; }
            }
        }
        for (int k0 = threadIdx.x; k0 < B * nt; k0 += 4 * SNN_GEN_THREADS) {
            float pv[4]; uint8_t sv[4];
            #pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int k = k0 + q * SNN_GEN_THREADS;
                pv[q] = k < B * nt ? __ldcg(pm + k) : 0.0f;
                sv[q] = k < B * nt ? __ldcg(st + k) : (uint8_t)0;
            }
            #pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int k = k0 + q * SNN_GEN_THREADS;
                if (k < B * nt) { pm_s[k] = pv[q]; st_s[k] = sv[q]; }
            }
        }
        for (int b = threadIdx.x; b < B; b += SNN_GEN_THREADS) sbw[b] = __ldcg(S.bits + ((size_t)wr * B + b) * S.nw + tile);
        __syncthreads();
    }
    // weight update from the eligibility of the previous step = p_plus (x) s_post + s_pre (x) p_minus
    if (C.rule == SNN_RULE_MSTDPET) {
        // learning.MSTDPET._connection_update (learning.py:2187-2249), batch size 1: the eligibility feeds a decaying
        // trace per synapse, the reward modulates the trace
        if (i < ns)
            for (int j = warp; j < nt; j += SNN_GEN_WARPS) {
                const bool ss = staged ? sp_s[lane] != 0 : __ldcg(sp + i) != 0;
                const bool tt = staged ? st_s[j] != 0 : __ldcg(st + j) != 0;
                const float ppv = staged ? pp_s[lane] : __ldcg(pp + i), pmv = staged ? pm_s[j] : __ldcg(pm + j);
                const float e = ppv * (tt ? 1.0f : 0.0f) + (ss ? 1.0f : 0.0f) * pmv;      // :2245-2247 of the previous step
                float et = __ldcg(C.e_trace + (size_t)i * nt + j) * C.e_trace_decay;   // :2229
                et = et + e / C.tc_e_trace;                                            // :2230
                C.e_trace[(size_t)i * nt + j] = et;
                // :2232-2238; a rate tensor is scaled per element, ((nu0 * dt) * reward) * e_trace left to right
                const float coef = SYN && C.nu0_t ? (syn_at(C.nu0_t, C.nu0_form, 0.0f, i, j, nt) * C.dt_scale) * C.reward : C.et_coef;
                float x = __ldcg(C.w + (size_t)i * nt + j) + coef * et;
                if (C.weight_decay != 0.0f) x = x * C.weight_decay;
                if (C.has_clamp) x = SYN ? clampf(x, syn_at(C.wmin_t, C.wmin_form, C.wmin, i, j, nt), syn_at(C.wmax_t, C.wmax_form, C.wmax, i, j, nt))
                                         : clampf(x, C.wmin, C.wmax);
                C.w[(size_t)i * nt + j] = x;
            }
    } else if (i < ns)
        for (int j = warp; j < nt; j += SNN_GEN_WARPS) {
            float upd = 0.0f;
            if (staged) {
                for (int b = 0; b < B; ++b) {
                    const bool ss = sp_s[b * 32 + lane] != 0, tt = st_s[b * nt + j] != 0;
                    if (!ss && !tt) continue;
                    const float e = pp_s[b * 32 + lane] * (tt ? 1.0f : 0.0f) + (ss ? 1.0f : 0.0f) * pm_s[b * nt + j];
                    upd = upd + C.reward * e;
                }
            } else {
                for (int b = 0; b < B; ++b) {
                    const bool ss = __ldcg(sp + (size_t)b * ns + i) != 0, tt = __ldcg(st + (size_t)b * nt + j) != 0;
                    if (!ss && !tt) continue;
                    const float e = __ldcg(pp + (size_t)b * ns + i) * (tt ? 1.0f : 0.0f) + (ss ? 1.0f : 0.0f) * __ldcg(pm + (size_t)b * nt + j);
                    upd = upd + C.reward * e;
                }
            }
            if (C.reduction == SNN_REDUCE_MEAN) upd = upd / Bf;
            float x = __ldcg(C.w + (size_t)i * nt + j) + (SYN ? syn_at(C.nu0_t, C.nu0_form, C.nu0, i, j, nt) : C.nu0) * upd;
            if (C.weight_decay != 0.0f) x = x * C.weight_decay;
            if (C.has_clamp) x = SYN ? clampf(x, syn_at(C.wmin_t, C.wmin_form, C.wmin, i, j, nt), syn_at(C.wmax_t, C.wmax_form, C.wmax, i, j, nt))
                                     : clampf(x, C.wmin, C.wmax);
            C.w[(size_t)i * nt + j] = x;
        }
    // P+ and the pre-synaptic spikes of this step for my rows; tile 0 also does P- and the post side
    if (i < ns)
        for (int b = warp; b < B; b += SNN_GEN_WARPS) {
            const size_t k = (size_t)b * ns + i;
            bool s;
            float p;
            if (staged) { s = (sbw[b] >> lane) & 1u; p = pp_s[b * 32 + lane]; }
            else { s = bit_of(S.bits + ((size_t)wr * B + b) * S.nw, i); p = __ldcg(pp + k); }
            M.pp[out][k] = mst_trace(p, C.p_plus_decay, C.a_plus, s);
            M.sp[out][k] = s ? 1 : 0;
        }
    if (tile == 0)
        for (size_t k = threadIdx.x; k < (size_t)B * nt; k += SNN_GEN_THREADS) {
            const int b = (int)(k / nt), jj = (int)(k - (size_t)b * nt);
            const bool s = bit_of(G.bits + ((size_t)wr * B + b) * G.nw, jj);
            M.pm[out][k] = mst_trace(__ldcg(pm + k), C.p_minus_decay, C.a_minus, s);
            M.st[out][k] = s ? 1 : 0;
        }
    if (staged) __syncthreads();   // the staging buffers belong to the CTA's next unit
}

// Ascending iterator over the set bits of row[lo, hi) (a bit row in shared memory, or in L2 when STAGED is off).
struct BitIter {
    const uint32_t *row;
    int w, wend, lo, hi;
    uint32_t cur;
    bool staged;
    __device__ __forceinline__ uint32_t load(int ww) const {
        uint32_t x = staged ? row[ww] : __ldcg(row + ww);
        const int base = ww * 32;
        if (base < lo) x &= 0xffffffffu << (lo - base);
        if (base + 32 > hi) x &= (hi - base >= 32) ? 0xffffffffu : ((1u << (hi - base)) - 1u);
        return x;
    }
    __device__ __forceinline__ void init(const uint32_t *r, int lo_, int hi_, bool st) {
        row = r; lo = lo_; hi = hi_; staged = st;
        w = lo >> 5; wend = (hi - 1) >> 5;
        cur = hi > lo ? load(w) : 0u;
        if (hi <= lo) w = wend = 0;
    }
    __device__ __forceinline__ int next() {
        while (cur == 0u) {
            if (w >= wend) return -1;
            ++w;
            cur = load(w);
        }
        const int idx = w * 32 + __ffs(cur) - 1;
        cur &= cur - 1;
        return idx;
    }
};

// One weight of PostPre / WeightDependentPostPre / Hebbian from its batch-reduced pre / post terms U / V, then the base
// class's decay and clamp (learning.py:457-497, 920-975, 1348-1380 on Conv2dConnection; :258-320, 717-791, 1186-1250 on
// LocalConnection2D; :87-104).  A term is applied when its nu is non-zero (Hebbian: always).
__device__ __forceinline__ float stdp_rule_apply(const snn_conn_t &C, float x, float U, float V, bool pre_on, bool post_on) {
    if (C.rule == SNN_RULE_WDEP_POSTPRE) {
        float upd = 0.0f;
        if (pre_on) upd = upd - (C.nu0 * U) * (x - C.wmin);
        if (post_on) upd = upd + (C.nu1 * V) * (C.wmax - x);
        x = x + upd;
    } else if (C.rule == SNN_RULE_HEBBIAN) {
        x = x + C.nu0 * U;
        x = x + C.nu1 * V;
    } else {
        if (pre_on) x = x - C.nu0 * U;
        if (post_on) x = x + C.nu1 * V;
    }
    if (C.weight_decay != 0.0f) x = x * C.weight_decay;
    if (C.has_clamp) x = clampf(x, C.wmin, C.wmax);
    return x;
}

// The source neuron of element (n', m) of a LocalConnection2D rule (snn_b200.h): the unfolded source at flat position
// (n' % P) * cin * K + m in [cin, P, K] order.  D3: a LocalConnection3D's (P and K over the depth axis too); without it the
// depth term is 1 and the depth fields are never read.
template <bool D3 = false>
__host__ __device__ __forceinline__ int local2d_rule_source(const snn_conn_t &C, int n, int m) {
    const int HW = C.hout * C.wout, KHW = C.kh * C.kw, K = (D3 ? C.kd : 1) * KHW, P = (D3 ? C.dout : 1) * HW;
    const int q = (n % P) * C.cin * K + m, ci = q / (P * K), r = q - ci * P * K, l = r / K, k = r - l * K;
    const int oz = D3 ? l / HW : 0, lr = l - oz * HW, kz = D3 ? k / KHW : 0, kr = k - kz * KHW;
    const int oy = lr / C.wout, ox = lr - oy * C.wout, ky = kr / C.kw, kx = kr - ky * C.kw;
    return ((ci * (D3 ? C.din : 1) + (D3 ? oz * C.sd + kz : 0)) * C.hin + oy * C.sh + ky) * C.win + ox * C.sw + kx;
}

// PostPre / WeightDependentPostPre / Hebbian on a LocalConnection2D (learning.py:258-320, 717-791, 1186-1250), and the
// decay of learning.NoOp.  Dense over w and spread over the grid (cta of ncta): element e = n' * cin * K + m takes
//   U = reduce_b x_tgt[b, n'] * s_src[b, src],  V = reduce_b s_tgt[b, n'] * x_src[b, src]   (src = local2d_rule_source)
// with the batch sum in ascending b, the terms of the silent samples skipped (they are exact zeros).  Traces are read
// from the layers' own arrays, framed by the grid barriers around the learning phase.  Every element is rewritten every
// step: the decay and the clamp reach all of w, and at B = 128 nearly every receptive field holds a pre-synaptic spike.
__device__ void phase3_local2d(const DevNet &N, int ci_, int cta, int ncta, int t) {
    const snn_conn_t &C = N.conns[ci_];
    const DevLayer &S = N.layers[C.src], &G = N.layers[C.tgt];
    const int B = N.B, ns = S.L.n, nt = G.L.n, Mw = C.cin * C.kh * C.kw;
    const size_t NW = (size_t)nt * Mw, start = (size_t)cta * SNN_GEN_THREADS + threadIdx.x, stride = (size_t)ncta * SNN_GEN_THREADS;
    if (!SNN_RULE_IS_STDP(C.rule)) {   // learning.NoOp: w *= weight_decay (learning.py:93-94), no clamp
        if (C.weight_decay != 0.0f)
            for (size_t e = start; e < NW; e += stride) C.w[e] = __ldcg(C.w + e) * C.weight_decay;
        return;
    }
    const bool hebb = C.rule == SNN_RULE_HEBBIAN;
    const bool pre_on = C.nu0 != 0.0f || hebb, post_on = C.nu1 != 0.0f || hebb;
    const int wr = t & 1;
    for (size_t e = start; e < NW; e += stride) {
        const int n = (int)(e / Mw), src = local2d_rule_source(C, n, (int)(e - (size_t)n * Mw));
        float U = 0.0f, V = 0.0f;
        for (int b = 0; b < B; ++b) {
            if (pre_on && bit_of(S.bits + ((size_t)wr * B + b) * S.nw, src)) U = U + __ldcg(G.L.x + (size_t)b * nt + n);
            if (post_on && bit_of(G.bits + ((size_t)wr * B + b) * G.nw, n)) V = V + __ldcg(S.L.x + (size_t)b * ns + src);
        }
        if (C.reduction == SNN_REDUCE_MEAN) { U = U / (float)B; V = V / (float)B; }
        C.w[e] = stdp_rule_apply(C, __ldcg(C.w + e), U, V, pre_on, post_on);
    }
}

// PostPre / WeightDependentPostPre / Hebbian on a LocalConnection3D (learning.py:322-388, 793-871, 1249-1314), and the
// decay of learning.NoOp.  Element (n', m) of w (flat n' * cin * K + m, source src = local2d_rule_source<true>) takes
//   U = reduce_b x_tgt[b, n'] * s_src[b, src],  V = reduce_b s_tgt[b, n'] * x_src[b, src]
// with the samples in ascending b from +0 and the terms of silent spikes skipped, as phase3_local2d.  Organised by target
// row rather than by element: a unit is one warp over SNN_LOCAL3D_EPL * 32 consecutive m of one row n', lane l holding
// m0 + 32 i + l.  x_tgt[b, n'] and s_tgt[b, n'] are then warp-uniform: the warp loads them for 32 samples at a time, and
// a sample whose x_tgt is zero (its U terms are +-0, which leave the +0-started sum as it is) or whose target is silent
// is skipped by the whole warp for U or V.  For cin = 1 neighbouring lanes read neighbouring source bits and traces.
// Traces are read from the layers' own arrays, framed by the grid barriers around the learning phase.
#define SNN_LOCAL3D_EPL 4
__device__ void phase3_local3d(const DevNet &N, int ci_, int cta, int ncta, int t) {
    const snn_conn_t &C = N.conns[ci_];
    const DevLayer &S = N.layers[C.src], &G = N.layers[C.tgt];
    const int B = N.B, ns = S.L.n, nt = G.L.n, Mw = C.cin * C.kd * C.kh * C.kw;
    if (!SNN_RULE_IS_STDP(C.rule)) {   // learning.NoOp: w *= weight_decay (learning.py:93-94), no clamp
        const size_t NW = (size_t)nt * Mw;
        if (C.weight_decay != 0.0f)
            for (size_t e = (size_t)cta * SNN_GEN_THREADS + threadIdx.x; e < NW; e += (size_t)ncta * SNN_GEN_THREADS)
                C.w[e] = __ldcg(C.w + e) * C.weight_decay;
        return;
    }
    const bool hebb = C.rule == SNN_RULE_HEBBIAN;
    const bool pre_on = C.nu0 != 0.0f || hebb, post_on = C.nu1 != 0.0f || hebb;
    const int wr = t & 1, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int segs = (Mw + 32 * SNN_LOCAL3D_EPL - 1) / (32 * SNN_LOCAL3D_EPL);
    const long long units = (long long)nt * segs;
    for (long long u = (long long)cta * SNN_GEN_WARPS + warp; u < units; u += (long long)ncta * SNN_GEN_WARPS) {
        const int n = (int)(u / segs), m0 = (int)(u - (long long)n * segs) * 32 * SNN_LOCAL3D_EPL + lane;
        int src[SNN_LOCAL3D_EPL];
        float U[SNN_LOCAL3D_EPL], V[SNN_LOCAL3D_EPL];
        #pragma unroll
        for (int i = 0; i < SNN_LOCAL3D_EPL; ++i) {
            const int m = m0 + 32 * i;
            src[i] = m < Mw ? local2d_rule_source<true>(C, n, m) : -1;
            U[i] = 0.0f; V[i] = 0.0f;
        }
        for (int b0 = 0; b0 < B; b0 += 32) {
            const int b = b0 + lane;
            float xt = 0.0f;
            bool st = false;
            if (b < B) {
                if (pre_on) xt = __ldcg(G.L.x + (size_t)b * nt + n);
                if (post_on) st = bit_of(G.bits + ((size_t)wr * B + b) * G.nw, n);
            }
            uint32_t um = __ballot_sync(0xffffffffu, xt != 0.0f), vm = __ballot_sync(0xffffffffu, st);
            while (um) {   // samples ascending
                const int q = __ffs(um) - 1;
                um &= um - 1;
                const float xb = __shfl_sync(0xffffffffu, xt, q);
                const uint32_t *sb = S.bits + ((size_t)wr * B + b0 + q) * S.nw;
                #pragma unroll
                for (int i = 0; i < SNN_LOCAL3D_EPL; ++i)
                    if (src[i] >= 0 && bit_of(sb, src[i])) U[i] = U[i] + xb;
            }
            while (vm) {
                const int q = __ffs(vm) - 1;
                vm &= vm - 1;
                const float *xs = S.L.x + (size_t)(b0 + q) * ns;
                #pragma unroll
                for (int i = 0; i < SNN_LOCAL3D_EPL; ++i)
                    if (src[i] >= 0) V[i] = V[i] + __ldcg(xs + src[i]);
            }
        }
        #pragma unroll
        for (int i = 0; i < SNN_LOCAL3D_EPL; ++i) {
            if (src[i] < 0) continue;
            float u1 = U[i], v1 = V[i];
            if (C.reduction == SNN_REDUCE_MEAN) { u1 = u1 / (float)B; v1 = v1 / (float)B; }
            const size_t e = (size_t)n * Mw + m0 + 32 * i;
            C.w[e] = stdp_rule_apply(C, __ldcg(C.w + e), u1, v1, pre_on, post_on);
        }
    }
}

// The updates a Conv3dConnection runs (snn_b200.h, snn_conv3d_rule_ok): learning.NoOp's w *= weight_decay
// (learning.py:93-94), and a zero-rate PostPre / WeightDependentPostPre's decay then clamp (:87-104).  Dense over w and
// spread over the grid (cta of ncta), like the conv2d NoOp branch.
__device__ void phase3_conv3d(const snn_conn_t &C, int cta, int ncta) {
    const size_t NW = (size_t)C.cout * C.cin * C.kd * C.kh * C.kw;
    const size_t start = (size_t)cta * SNN_GEN_THREADS + threadIdx.x, stride = (size_t)ncta * SNN_GEN_THREADS;
    const bool clamp = C.rule != SNN_RULE_NOOP && C.has_clamp;
    if (C.weight_decay == 0.0f && !clamp) return;
    for (size_t e = start; e < NW; e += stride) {
        float x = __ldcg(C.w + e);
        if (C.weight_decay != 0.0f) x = x * C.weight_decay;
        if (clamp) x = clampf(x, C.wmin, C.wmax);
        C.w[e] = x;
    }
}

// PostPre / WeightDependentPostPre / Hebbian on a Conv1dConnection (learning.py:422-455, 873-918, 1316-1346), and the
// decay of learning.NoOp.  Element e = co * cin * kw + m takes (snn_b200.h)
//   U = reduce_b sum_l' x_tgt[b, co, l'] * s_src[b, src(l', m)],  V = reduce_b sum_l' s_tgt[b, co, l'] * x_src[b, src(l', m)]
// where src is the source neuron the reference's reshape of the unfolded source pairs with target position l'.  Along
// l' that pairing keeps kk' = m % kw and advances the unfolded row l by cin (wrapping into the next channel c), so it is
// stepped, not divided out.  One warp per group of 32 / g elements, g lanes per element over the samples (g = B rounded
// up to a power of two, at most 32): each lane builds its sample's partial sums over l' ascending, visiting the target
// bits a word at a time and skipping the terms of silent spikes; the partials then join in ascending b through
// shuffles, g samples at a time.  Traces are read from the layers' own arrays, framed by the grid barriers around the
// learning phase.
__device__ void phase3_conv1d(const DevNet &N, int ci_, int cta, int ncta, int t) {
    const snn_conn_t &C = N.conns[ci_];
    const DevLayer &S = N.layers[C.src], &G = N.layers[C.tgt];
    const int B = N.B, ns = S.L.n, nt = G.L.n, Mw = C.cin * C.kw, L = C.wout, NW = C.cout * Mw;
    if (!SNN_RULE_IS_STDP(C.rule)) {   // learning.NoOp: w *= weight_decay (learning.py:93-94), no clamp
        if (C.weight_decay != 0.0f)
            for (int e = cta * SNN_GEN_THREADS + threadIdx.x; e < NW; e += ncta * SNN_GEN_THREADS) C.w[e] = __ldcg(C.w + e) * C.weight_decay;
        return;
    }
    const bool hebb = C.rule == SNN_RULE_HEBBIAN;
    const bool pre_on = C.nu0 != 0.0f || hebb, post_on = C.nu1 != 0.0f || hebb;
    const int wr = t & 1, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int g = 1;
    while (g < B && g < 32) g <<= 1;
    const int epw = 32 / g, base = lane & ~(g - 1), sub = lane - base, LK = L * C.kw;
    for (int e0 = (cta * SNN_GEN_WARPS + warp) * epw; e0 < NW; e0 += ncta * SNN_GEN_WARPS * epw) {
        const int e = e0 + lane / g;
        const bool ok = e < NW;
        const int co = ok ? e / Mw : 0, m = ok ? e - co * Mw : 0;
        const int c0 = m / LK, r0 = m - c0 * LK, l0 = r0 / C.kw, off = r0 - l0 * C.kw - C.pw;   // the pairing at l' = 0
        float U = 0.0f, V = 0.0f;
        for (int bq = 0; bq < B; bq += g) {
            const int b = bq + sub;
            float u1 = 0.0f, v1 = 0.0f;
            if (ok && b < B) {
                const uint32_t *sb = S.bits + ((size_t)wr * B + b) * S.nw, *gb = G.bits + ((size_t)wr * B + b) * G.nw;
                const float *xt = G.L.x + (size_t)b * nt + (size_t)co * L, *xs = S.L.x + (size_t)b * ns;
                int c = c0, l = l0, cw = -1;
                uint32_t cword = 0u;   // the source bit word last read (word cw)
                for (int lq = 0; lq < L; lq += 32) {
                    const int cnt = min(32, L - lq), bit0 = co * L + lq, w0 = bit0 >> 5, sft = bit0 & 31;
                    uint32_t tw = 0u;   // target spikes of l' in [lq, lq + cnt)
                    if (post_on) {
                        const uint32_t lo = __ldcg(gb + w0), hi = sft + cnt > 32 ? __ldcg(gb + w0 + 1) : 0u;
                        tw = __funnelshift_r(lo, hi, sft) & (cnt >= 32 ? 0xffffffffu : ((1u << cnt) - 1u));
                    }
                    for (int q = 0; q < cnt; ++q) {
                        const int pos = l * C.sw + off;
                        if (pos >= 0 && pos < C.win) {
                            const int src = c * C.win + pos;
                            if (pre_on) {
                                if ((src >> 5) != cw) { cw = src >> 5; cword = __ldcg(sb + cw); }
                                if ((cword >> (src & 31)) & 1u) u1 = u1 + __ldcg(xt + lq + q);
                            }
                            if ((tw >> q) & 1u) v1 = v1 + __ldcg(xs + src);
                        }
                        l += C.cin;
                        while (l >= L) { l -= L; ++c; }
                    }
                }
            }
            const int nb = min(g, B - bq);
            for (int q = 0; q < nb; ++q) {
                const float uq = __shfl_sync(0xffffffffu, u1, base + q), vq = __shfl_sync(0xffffffffu, v1, base + q);
                U = U + uq;
                V = V + vq;
            }
        }
        if (ok && sub == 0) {
            if (C.reduction == SNN_REDUCE_MEAN) { U = U / (float)B; V = V / (float)B; }
            C.w[e] = stdp_rule_apply(C, __ldcg(C.w + e), U, V, pre_on, post_on);
        }
    }
}

// learning.MSTDP._conv2d_connection_update (learning.py:1942-2015) with a per-sample eligibility
// (SURVEY.md §0.8), PostPre / WeightDependentPostPre / Hebbian on a Conv2dConnection, and the decay-only
// update of a conv connection without a rule (learning.NoOp).  Called once per CTA and step: every loop is
// spread over the whole grid (cta of ncta).
__device__ void phase3_conv(const DevNet &N, int ci_, int cta, int ncta, int t, const GenSmem &GS) {
    const snn_conn_t &C = N.conns[ci_];
    const DevMstdp &M = N.mst[ci_];
    const DevLayer &S = N.layers[C.src], &G = N.layers[C.tgt];
    const int B = N.B, ns = S.L.n, nt = G.L.n;
    const int KK = C.kh * C.kw, K = C.cin * KK, L = C.hout * C.wout, NWT = C.cout * K;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const size_t start = (size_t)cta * SNN_GEN_THREADS + threadIdx.x, stride = (size_t)ncta * SNN_GEN_THREADS;
    if (SNN_RULE_IS_STDP(C.rule)) {
        // PostPre / WeightDependentPostPre / Hebbian on the im2col views (learning.py:457-497, 920-975, 1348-1380):
        // per filter tap (co, k) the inner sum runs over the output positions (ascending) of one sample, the outer
        // one over the samples (ascending) — the oracle's order.  Traces are read from the layers' own arrays:
        // the grid barriers before and after the learning phase frame them.
        const bool hebb = C.rule == SNN_RULE_HEBBIAN;
        const bool pre_on = C.nu0 != 0.0f || hebb, post_on = C.nu1 != 0.0f || hebb;
        const int wr = t & 1;
        for (size_t e = start; e < (size_t)NWT; e += stride) {
            const int co = (int)(e / K), k = (int)(e - (size_t)co * K);
            const int ci = k / KK, kk = k - ci * KK, ky = kk / C.kw, kx = kk - ky * C.kw;
            float U = 0.0f, V = 0.0f;
            for (int b = 0; b < B; ++b) {
                const uint32_t *sb = S.bits + ((size_t)wr * B + b) * S.nw, *gb = G.bits + ((size_t)wr * B + b) * G.nw;
                float u1 = 0.0f, v1 = 0.0f;
                for (int oy = 0; oy < C.hout; ++oy) {
                    const int iy = oy * C.sh - C.ph + ky;
                    if (iy < 0 || iy >= C.hin) continue;
                    for (int ox = 0; ox < C.wout; ++ox) {
                        const int ix = ox * C.sw - C.pw + kx;
                        if (ix < 0 || ix >= C.win) continue;
                        const int src = (ci * C.hin + iy) * C.win + ix, tgt = co * L + oy * C.wout + ox;
                        if (pre_on && bit_of(sb, src)) u1 = u1 + __ldcg(G.L.x + (size_t)b * nt + tgt);
                        if (post_on && bit_of(gb, tgt)) v1 = v1 + __ldcg(S.L.x + (size_t)b * ns + src);
                    }
                }
                U = U + u1; V = V + v1;
            }
            if (C.reduction == SNN_REDUCE_MEAN) { U = U / (float)B; V = V / (float)B; }
            C.w[e] = stdp_rule_apply(C, __ldcg(C.w + e), U, V, pre_on, post_on);
        }
        return;
    }
    if (C.rule != SNN_RULE_MSTDP) {  // learning.NoOp: w *= weight_decay (learning.py:93-94), no clamp
        if (C.rule == SNN_RULE_NOOP && C.weight_decay != 0.0f)
            for (size_t k = start; k < (size_t)NWT; k += stride) C.w[k] = __ldcg(C.w + k) * C.weight_decay;
        return;
    }
    const int in = (t + N.T) & 1, out = in ^ 1, wr = t & 1;
    const float *pp = M.pp[in], *pm = M.pm[in], *el = M.el[in];
    // w += nu0 * sum_b reward * eligibility(t-1)  (:1973-1974), then decay / clamp (learning.py:87-104).
    // One warp per filter tap: the lanes fetch 32 samples' eligibilities at once, the sum itself stays serial
    // in ascending b (shuffles, no memory latency in the chain).
    for (int k = cta * SNN_GEN_WARPS + warp; k < NWT; k += ncta * SNN_GEN_WARPS) {
        float upd = 0.0f;
        for (int bq = 0; bq < B; bq += 32) {
            const float val = (bq + lane < B) ? __ldcg(el + (size_t)(bq + lane) * NWT + k) : 0.0f;
            const int m = min(32, B - bq);
            for (int q = 0; q < m; ++q) upd = upd + C.reward * __shfl_sync(0xffffffffu, val, q);
        }
        if (lane == 0) {
            float x = __ldcg(C.w + k) + C.nu0 * upd;
            if (C.weight_decay != 0.0f) x = x * C.weight_decay;
            if (C.has_clamp) x = clampf(x, C.wmin, C.wmax);
            C.w[k] = x;
        }
    }
    // P+ (trace image of the source), P- (:1999-2003); four elements per thread in flight
    {
        const size_t tot = (size_t)B * ns;
        for (size_t k0 = start; k0 < tot; k0 += 4 * stride) {
            float pv[4]; bool sv[4];
            #pragma unroll
            for (int q = 0; q < 4; ++q) {
                const size_t k = k0 + q * stride;
                pv[q] = 0.0f; sv[q] = false;
                if (k < tot) {
                    const int b = (int)(k / ns), i = (int)(k - (size_t)b * ns);
                    pv[q] = __ldcg(pp + k);
                    sv[q] = bit_of(S.bits + ((size_t)wr * B + b) * S.nw, i);
                }
            }
            #pragma unroll
            for (int q = 0; q < 4; ++q) {
                const size_t k = k0 + q * stride;
                if (k < tot) M.pp[out][k] = mst_trace(pv[q], C.p_plus_decay, C.a_plus, sv[q]);
            }
        }
    }
    {
        const size_t tot = (size_t)B * nt;
        for (size_t k0 = start; k0 < tot; k0 += 4 * stride) {
            float pv[4]; bool sv[4];
            #pragma unroll
            for (int q = 0; q < 4; ++q) {
                const size_t k = k0 + q * stride;
                pv[q] = 0.0f; sv[q] = false;
                if (k < tot) {
                    const int b = (int)(k / nt), jj = (int)(k - (size_t)b * nt);
                    pv[q] = __ldcg(pm + k);
                    sv[q] = bit_of(G.bits + ((size_t)wr * B + b) * G.nw, jj);
                }
            }
            #pragma unroll
            for (int q = 0; q < 4; ++q) {
                const size_t k = k0 + q * stride;
                if (k < tot) M.pm[out][k] = mst_trace(pv[q], C.p_minus_decay, C.a_minus, sv[q]);
            }
        }
    }
    // eligibility(t)[b,co,k] = sum_l s_post[b,co,l] * P+col[b,k,l]  +  sum_l P-[b,co,l] * s_pre_col[b,k,l]
    // (:2005-2009), l = (oy, ox) ascending, with the UPDATED traces (recomputed here from slot `in`).
    // Only spiking positions contribute, so each sum walks the set bits of the sample's target (source) bit row
    // inside channel co (ci) in ascending order — the same terms in the same order as the dense double loop.
    // Unit = (sample, group of output channels); the sample's two bit rows are staged in shared memory.
    {
        // output channels per unit: about one (channel, tap) element per thread, and few enough channels for their
        // P- rows of the sample ([channels][L] floats) to be staged in the 32 KB accumulator region
        const bool stage_pm = L <= SNN_GEN_WARPS * 32 * 32;
        const int cpc = stage_pm ? min(max(1, SNN_GEN_THREADS / K), (SNN_GEN_WARPS * 32 * 32) / L) : max(1, SNN_GEN_THREADS / K);
        const int nch = (C.cout + cpc - 1) / cpc;
        const bool staged = S.nw + G.nw <= SNN_CONV_STAGE_WORDS;
        uint32_t *sb_s = (uint32_t *)GS.xs, *gb_s = (uint32_t *)GS.xs + S.nw;
        float *pm_s = GS.acc;
        // the sample's source spikes as an ascending list of (src << 16 | iy << 8 | ix), decoded once per unit instead
        // of once per (filter tap, spike); it shares the 16 KB region with the two bit rows
        uint32_t *slist = (uint32_t *)GS.xs + S.nw + G.nw;
        const int slist_cap = staged ? SNN_CONV_STAGE_WORDS - S.nw - G.nw - (C.cin + 2) : 0;
        int32_t *seg = (int32_t *)(slist + (slist_cap > 0 ? slist_cap : 0));   // [cin + 1] first list entry of every input channel
        const bool listed = staged && ns <= 65535 && C.hin <= 256 && C.win <= 256 && slist_cap >= ns;
        const bool unit_stride = C.sh == 1 && C.sw == 1;
        for (int u = cta; u < B * nch; u += ncta) {
            const int b = u / nch, ch = u - b * nch;
            const int co0 = ch * cpc, co1 = min(C.cout, co0 + cpc);
            const uint32_t *sbg = S.bits + ((size_t)wr * B + b) * S.nw, *gbg = G.bits + ((size_t)wr * B + b) * G.nw;
            const float *ppb = pp + (size_t)b * ns, *pmb = pm + (size_t)b * nt;
            if (staged || stage_pm) __syncthreads();
            if (staged) {
                for (int k = threadIdx.x; k < S.nw; k += SNN_GEN_THREADS) sb_s[k] = __ldcg(sbg + k);
                for (int k = threadIdx.x; k < G.nw; k += SNN_GEN_THREADS) gb_s[k] = __ldcg(gbg + k);
            }
            if (stage_pm) {   // P- of the unit's channels, eight loads in flight per thread
                const int tot = (co1 - co0) * L;
                const float *src = pmb + (size_t)co0 * L;
                for (int k0 = threadIdx.x; k0 < tot; k0 += 8 * SNN_GEN_THREADS) {
                    float pv8[8];
                    #pragma unroll
                    for (int q = 0; q < 8; ++q) pv8[q] = k0 + q * SNN_GEN_THREADS < tot ? __ldcg(src + k0 + q * SNN_GEN_THREADS) : 0.0f;
                    #pragma unroll
                    for (int q = 0; q < 8; ++q)
                        if (k0 + q * SNN_GEN_THREADS < tot) pm_s[k0 + q * SNN_GEN_THREADS] = pv8[q];
                }
            }
            if (staged || stage_pm) __syncthreads();
            const uint32_t *sb = staged ? sb_s : sbg, *gb = staged ? gb_s : gbg;
            if (listed) {
                if (warp == 0) {   // ordered compaction of the set bits, 32 words at a time
                    int n_ent = 0;
                    for (int w0 = 0; w0 < S.nw; w0 += 32) {
                        uint32_t mine = w0 + lane < S.nw ? sb_s[w0 + lane] : 0u;
                        const int cnt = __popc(mine);
                        int pre = cnt;
                        #pragma unroll
                        for (int o = 1; o < 32; o <<= 1) {
                            const int v = __shfl_up_sync(0xffffffffu, pre, o);
                            if (lane >= o) pre += v;
                        }
                        int q = n_ent + pre - cnt;
                        n_ent += __shfl_sync(0xffffffffu, pre, 31);
                        while (mine) {
                            const int src = (w0 + lane) * 32 + __ffs(mine) - 1;
                            mine &= mine - 1;
                            const int r = src % (C.hin * C.win), iy = r / C.win, ix = r - iy * C.win;
                            slist[q++] = ((uint32_t)src << 16) | ((uint32_t)iy << 8) | (uint32_t)ix;
                        }
                    }
                    __syncwarp();
                    // seg[c] = number of entries whose source index lies below channel c
                    for (int c = lane; c <= C.cin; c += 32) {
                        const uint32_t lim = (uint32_t)(c * C.hin * C.win);
                        int lo = 0, hi = n_ent;
                        while (lo < hi) { const int mid = (lo + hi) >> 1; if ((slist[mid] >> 16) < lim) lo = mid + 1; else hi = mid; }
                        seg[c] = lo;
                    }
                }
                __syncthreads();
            }
            for (int e = threadIdx.x; e < (co1 - co0) * K; e += SNN_GEN_THREADS) {
                const int co = co0 + e / K, k = e - (co - co0) * K;
                const int ci = k / KK, kk = k - ci * KK, ky = kk / C.kw, kx = kk - ky * C.kw;
                float s1 = 0.0f, s2 = 0.0f;
                BitIter it;
                // post-synaptic spikes of channel co
                it.init(gb, co * L, (co + 1) * L, staged);
                for (;;) {
                    const int tgt = it.next();
                    if (tgt < 0) break;
                    const int l = tgt - co * L, oy = l / C.wout, ox = l - oy * C.wout;
                    const int iy = oy * C.sh - C.ph + ky, ix = ox * C.sw - C.pw + kx;
                    if (iy < 0 || iy >= C.hin || ix < 0 || ix >= C.win) continue;
                    const int src = (ci * C.hin + iy) * C.win + ix;
                    const bool ss = ((staged ? sb[src >> 5] : __ldcg(sb + (src >> 5))) >> (src & 31)) & 1u;
                    s1 = s1 + mst_trace(__ldcg(ppb + src), C.p_plus_decay, C.a_plus, ss);
                }
                // pre-synaptic spikes of channel ci
                if (listed) {
                    const int e1 = seg[ci + 1];
                    for (int q = seg[ci]; q < e1; ++q) {
                        const uint32_t ent = slist[q];
                        const int ty = (int)((ent >> 8) & 255u) + C.ph - ky, tx = (int)(ent & 255u) + C.pw - kx;
                        if (ty < 0 || tx < 0) continue;
                        int oy = ty, ox = tx;
                        if (!unit_stride) {
                            oy = ty / C.sh; ox = tx / C.sw;
                            if (oy * C.sh != ty || ox * C.sw != tx) continue;
                        }
                        if (oy >= C.hout || ox >= C.wout) continue;
                        const int tgt = co * L + oy * C.wout + ox;
                        const float pv = stage_pm ? pm_s[tgt - co0 * L] : __ldcg(pmb + tgt);
                        const bool ts = (gb[tgt >> 5] >> (tgt & 31)) & 1u;
                        s2 = s2 + mst_trace(pv, C.p_minus_decay, C.a_minus, ts);
                    }
                    M.el[out][(size_t)b * NWT + (size_t)co * K + k] = s1 + s2;
                    continue;
                }
                // ... the same walk straight off the bit row (shapes the list does not cover), four trace loads in flight
                const int cbase = ci * C.hin * C.win;
                it.init(sb, cbase, cbase + C.hin * C.win, staged);
                bool done = false;
                while (!done) {
                    int tg[4];
                    #pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        tg[q] = -1;
                        if (done) continue;
                        const int src = it.next();
                        if (src < 0) { done = true; continue; }
                        const int r = src - cbase, iy = r / C.win, ix = r - iy * C.win;
                        const int ty = iy + C.ph - ky, tx = ix + C.pw - kx;
                        if (ty < 0 || tx < 0) continue;
                        const int oy = ty / C.sh, ox = tx / C.sw;
                        if (oy * C.sh != ty || ox * C.sw != tx || oy >= C.hout || ox >= C.wout) continue;
                        tg[q] = co * L + oy * C.wout + ox;
                    }
                    float pv[4];
                    #pragma unroll
                    for (int q = 0; q < 4; ++q) pv[q] = tg[q] >= 0 ? (stage_pm ? pm_s[tg[q] - co0 * L] : __ldcg(pmb + tg[q])) : 0.0f;
                    #pragma unroll
                    for (int q = 0; q < 4; ++q)
                        if (tg[q] >= 0) {
                            const bool ts = ((staged ? gb[tg[q] >> 5] : __ldcg(gb + (tg[q] >> 5))) >> (tg[q] & 31)) & 1u;
                            s2 = s2 + mst_trace(pv[q], C.p_minus_decay, C.a_minus, ts);
                        }
                }
                M.el[out][(size_t)b * NWT + (size_t)co * K + k] = s1 + s2;
            }
        }
        if (staged || stage_pm) __syncthreads();
    }
}

// learning.NoOp on a SparseConnection: every stored value *= weight_decay (learning.py:93-94), no clamp; spread over the
// grid (cta of ncta).
__device__ __forceinline__ void decay_sparse(const snn_conn_t &C, int cta, int ncta) {
    if (C.rule != SNN_RULE_NOOP || C.weight_decay == 0.0f || C.weight_decay == 1.0f) return;
    for (size_t k = (size_t)cta * SNN_GEN_THREADS + threadIdx.x; k < (size_t)C.nnz; k += (size_t)ncta * SNN_GEN_THREADS)
        C.w[k] = __ldcg(C.w + k) * C.weight_decay;
}

// Conv2dConnection.normalize (topology.py:824-837): every (out, in) filter scaled to sum `norm`
// (plain sum in ascending order; no guard against a zero sum, like the reference).
// Conv2dConnection.normalize (topology.py:824-837) and Conv3dConnection.normalize (:1004-1018): every (out, in) filter of
// KK taps (kh * kw, or kd * kh * kw) scaled by norm / its sum.
__device__ void normalize_conv_item(const snn_conn_t &C, int KK, int tile, int ntiles) {
    const int F = C.cout * C.cin;
    for (int f = tile * SNN_GEN_THREADS + threadIdx.x; f < F; f += ntiles * SNN_GEN_THREADS) {
        float tot = 0.0f;
        for (int k = 0; k < KK; ++k) tot = tot + C.w[(size_t)f * KK + k];
        const float fac = C.norm / tot;
        for (int k = 0; k < KK; ++k) C.w[(size_t)f * KK + k] = C.w[(size_t)f * KK + k] * fac;
    }
}

// LocalConnection2D.normalize (topology.py:1748-1759) and LocalConnection3D.normalize (:1898-1909): w viewed as
// [cin * n, K], every row scaled by norm / its sum (sum in ascending k; `norm / sum` is torch's reciprocal(sum) * norm).
// No guard against a zero sum, like the reference: such a row becomes inf / NaN.
__device__ void normalize_local2d_item(const snn_conn_t &C, int rows, int K, int tile, int ntiles) {
    for (int r = tile * SNN_GEN_THREADS + threadIdx.x; r < rows; r += ntiles * SNN_GEN_THREADS) {
        float *w = C.w + (size_t)r * K;
        float tot = 0.0f;
        for (int k = 0; k < K; ++k) tot = tot + w[k];
        const float fac = (1.0f / tot) * C.norm;
        for (int k = 0; k < K; ++k) w[k] = w[k] * fac;
    }
}

// Connection masks (Network.run(..., masks=...), network.py:449 -> AbstractConnection.update, topology.py:127-131): the
// masked weights of this column tile are zero after every step's update.
__device__ void mask_tile(const snn_conn_t &C, int ns, int nt, int tile) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int j = tile * SNN_TILE + lane;
    if (j < nt)
        for (int i = warp; i < ns; i += SNN_GEN_WARPS) {
            const size_t k = (size_t)i * nt + j;
            if (C.mask[k]) C.w[k] = 0.0f;
        }
    __syncthreads();
}

// normalize(): Connection.normalize (topology.py:383-392) / AbstractFeature.normalize
// (topology_features.py:250-266) on one tile; row chunking as documented in snn_b200.h.
// WN: the connection may carry a per-target norm tensor or normalise every step (snn_b200.h SNN_CONN_WNORM); the
// factor then follows the reference's rounding for that form, and w is read through L2, because inside a window other
// CTAs wrote it since the last grid barrier.  Without WN the function is the scalar end-of-window normalize.
template <bool WN = false>
__device__ void normalize_tile(const snn_conn_t &C, int ns, int nt, int tile, float *s_part) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int j = tile * SNN_TILE + lane;
    const bool valid = j < nt;
    const int chunk = (ns + SNN_NORM_CHUNKS - 1) / SNN_NORM_CHUNKS;
    __syncthreads();
    for (int c = warp; c < SNN_NORM_CHUNKS; c += SNN_GEN_WARPS) {
        float part = 0.0f;
        const int i1 = min((c + 1) * chunk, ns);
        if (valid)
            for (int i = c * chunk; i < i1; ++i) {
                const float x = WN ? __ldcg(C.w + (size_t)i * nt + j) : C.w[(size_t)i * nt + j];
                part = part + (C.norm_abs ? fabsf(x) : x);
            }
        s_part[c * 32 + lane] = part;
    }
    __syncthreads();
    if (warp == 0) {
        float tot = 0.0f;
        for (int c = 0; c < SNN_NORM_CHUNKS; ++c) tot = tot + s_part[c * 32 + lane];
        if (tot == 0.0f) tot = 1.0f;
        if (WN && C.norm_t) s_part[SNN_NORM_CHUNKS * 32 + lane] = (valid ? C.norm_t[j] : 0.0f) / tot;   // Tensor / Tensor
        else if (WN && C.norm_step) s_part[SNN_NORM_CHUNKS * 32 + lane] = (1.0f / tot) * C.norm;   // float / Tensor
        else s_part[SNN_NORM_CHUNKS * 32 + lane] = C.norm / tot;
    }
    __syncthreads();
    const float f = s_part[SNN_NORM_CHUNKS * 32 + lane];
    if (valid)
        for (int i = warp; i < ns; i += SNN_GEN_WARPS)
            C.w[(size_t)i * nt + j] = (WN ? __ldcg(C.w + (size_t)i * nt + j) : C.w[(size_t)i * nt + j]) * f;
    __syncthreads();
}


}  // namespace
