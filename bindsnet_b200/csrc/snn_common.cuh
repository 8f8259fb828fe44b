// snn_common.cuh — device-side helpers shared by the window kernels.
//
// Arithmetic contract: every floating-point operation below is a single IEEE fp32 rounding, in
// the order the reference's ATen ops apply them (the library is compiled with --fmad=false, so
// the compiler never contracts a*b+c).  Where the reference leaves a summation order to ATen
// the kernels sum in ascending index order, like oracle/snn_oracle.c, so kernel and oracle
// agree bit for bit.
#pragma once

#ifdef SNN_EMU   // tests/emu: the same sources compiled for the host on a small CUDA-model emulation (test infrastructure)
#include "cuda_emu.h"
#else
#include <cuda_runtime.h>
#endif
#include <stdint.h>

#include "../../include/snn_b200.h"

// Kernel launches and statically sized __shared__ arrays of the small kernels (snn_ops.cu, snn_encode.cu, snn_readout.cu)
// go through these two macros so that tests/emu can run the same sources on its CUDA-model emulation.
#ifdef SNN_EMU
#define SNN_LAUNCH(kernel, grid, block, smem, stream, ...) emu::launch((grid), (block), (size_t)(smem), [&]() { kernel(__VA_ARGS__); })
#define SNN_SHARED(type, name, count) type *name = (type *)emu::static_shared(sizeof(type) * (size_t)(count))
#define SNN_SHARED2(type, name, rows, cols) type(*name)[cols] = (type(*)[cols])emu::static_shared(sizeof(type) * (size_t)(rows) * (cols))
#define SNN_DYN_SHARED(type, name) type *name = (type *)emu::tls_cta->dyn_smem
#else
#define SNN_LAUNCH(kernel, grid, block, smem, stream, ...) kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__)
#define SNN_SHARED(type, name, count) __shared__ type name[count]
#define SNN_SHARED2(type, name, rows, cols) __shared__ type name[rows][cols]
#define SNN_DYN_SHARED(type, name) extern __shared__ type name[]
#endif

#define SNN_TILE 32          // neurons (columns) per work item: one warp lane per column
#define SNN_GEN_THREADS 256  // generic kernel: 8 warps per CTA
#define SNN_GEN_WARPS (SNN_GEN_THREADS / 32)

// The generic window's barrier block: SNN_BAR_WORDS counter words, then three spike-count slots per layer (DevLayer::spc),
// all zeroed before every launch.
#define SNN_BAR_WORDS 96
#define SNN_BAR_ZERO_WORDS (SNN_BAR_WORDS + 3 * SNN_MAX_LAYERS)

struct DevLayer {
    snn_layer_t L;
    uint32_t *bits;             // [2][B][nw]  bit-packed spikes, slot t&1 holds s(t)
    uint32_t *candbits;         // [B][nw]     DC one_spike: threshold crossers of this step
    unsigned long long *keys;   // [2][B]      DC one_spike: arg-max tie-break keys
    float *xpub;                // [2][B][n]   trace published for STDP readers (slot t&1), or NULL
    float *thdec;               // [2][n]      DC: the decayed adaptive threshold step t used (slot t&1)
    int32_t *thcnt;             // [3][n]      DC: threshold crossers of step t summed over the batch (slot t%3)
    uint32_t *anyf;             // [3][B]      wide source layers (nw > 32) of dense connections: non-zero iff the sample spiked
                                //             in step t (slot t%3) — lets a gather skip an all-zero bit row without reading it
    int32_t *spc;               // [3]         source of a MeanFieldConnection: the spikes of step t counted over the
                                //             batch and the layer (slot t%3); NULL for every other layer
    int32_t nw;                 // ceil(n / 32)
    int32_t item0;              // first work-item index of this layer
};

// State of an MSTDP rule, double-buffered: step t reads slot (t + T) & 1 and writes the other one, so
// that no thread overwrites a value another one still needs in the same step; slot 0 is the caller's
// tensors (snn_conn_t::p_plus ...), slot 1 lives in the workspace.
struct DevMstdp {
    float *pp[2], *pm[2], *el[2];
    uint8_t *sp[2], *st[2];
};

// A SparseConnection (SNN_CONN_SPARSE) in the generic window: its target columns are cut into blocks of `bw` columns;
// off[i * (nb + 1) + k] is the first CSR position of row i whose column is >= k * bw (k = nb: the row's end), built
// from the pattern once per window; out holds the connection's gathered input of the current step.
struct DevSparse {
    int32_t *off;               // [n_src][nb + 1]
    float *out;                 // [B][n_tgt]
    int32_t bw, nb;             // columns per block, blocks
    int32_t first;              // first gather unit of this connection
};

// Columns per block of a sparse connection's gather: 1024 (the per-warp accumulator in shared memory) unless the
// (block, 8-sample chunk) units would leave most of a 132-SM grid idle.  A unit's cost is set by the spiking rows it
// visits, not by the block width (each spiking row is visited once per block), so blocks are only narrowed until
// there are about 200 units; never below 128 columns, and never so narrow that the offset table (n_src x (blocks + 1)
// int32) outgrows max(16 MiB, twice the CSR itself).
__host__ __device__ inline int sparse_block_width(int n_src, int n_tgt, int B, int nnz) {
    const double cap = 16.0 * nnz > 16777216.0 ? 16.0 * nnz : 16777216.0;
    int bw = 1024;
    while (bw > 128 && (long long)((n_tgt + bw - 1) / bw) * ((B + 7) / 8) < 200 &&
           4.0 * n_src * ((n_tgt + bw / 2 - 1) / (bw / 2) + 1) <= cap)
        bw >>= 1;
    return bw;
}

// The slot bitmaps of an averaged MCC PostPre (snn_b200.h SNN_RULE_AVG), double-buffered like DevMstdp: step t reads slot
// (t + T) & 1 and writes the other one, slot 0 is the caller's avg_rows / avg_cols, slot 1 lives in the workspace.  Every
// unit of the learning phase reads a slot's previous bitmap while the one that owns its word writes the new one.
struct DevAvg {
    uint32_t *rows[2], *cols[2];
};
// The plan (after snn_api.cu's strip) runs a connection's MCC PostPre with averaging: the library clears avg_k on every
// other MCC PostPre connection, and no other rule reads the field.
__host__ __device__ __forceinline__ bool snn_is_avg(const snn_conn_t &C) { return C.rule == SNN_RULE_MCC_POSTPRE && C.avg_k > 0; }

struct DevNet {
    int32_t n_layers, n_conns, learning, T, B, normalize, total_items, any_one_spike;
    int32_t any_mask;             // some connection carries a mask (Network.run(..., masks=...))
    int32_t one_step;             // Network.run(one_step=True): layers in insertion order, inputs from current spikes
    uint32_t seed, step_offset;
    int32_t nch, cs;              // phases 1 / 2: sample chunks per tile, samples per chunk
    int32_t p3_total;             // phase 3: number of work units
    int32_t p3_first[SNN_MAX_CONNS], p3_rc[SNN_MAX_CONNS];   // first unit / row chunks per tile of every connection
    int32_t *err;               // device error flags (may be NULL)
    long long *prof;            // profiling only (env SNN_B200_GPROF): [grid][8] phase cycles of thread 0
    unsigned int *bar;          // [0] arrival count, [32] generation, [64] abort
    DevLayer layers[SNN_MAX_LAYERS];
    snn_conn_t conns[SNN_MAX_CONNS];
    DevMstdp mst[SNN_MAX_CONNS];
    int32_t sp_units;             // sparse gather units of a step (0: the plan has no SparseConnection)
    DevSparse sp[SNN_MAX_CONNS];
    int32_t any_feat;             // some MCC connection carries Probability / Mask / Intensity features
    int32_t any_pool;             // some connection is of a kind snn_pool_inst_kind names, or some layer is an
                                  // SNN_NODE_SUBIF / SNN_NODE_PASSTHROUGH one: the plan runs the POOL instantiation
    float *pool_r1[SNN_MAX_CONNS];   // MaxPool2d / MaxPoo3dConnection: the workspace slot of its rates (pool_rate_slot)
    DevAvg avg[SNN_MAX_CONNS];    // MCC PostPre with averaging (snn_is_avg)
    int32_t any_avg;              // some connection is one: the plan runs an AVG instantiation
    int32_t any_wn;               // some dense / MCC connection carries SNN_CONN_WNORM: the plan runs a WN instantiation
    int32_t wn_units;             // per-step normalisation units of a step (a column tile of a step-normalised Weight)
    int32_t wn_first[SNN_MAX_CONNS];   // first such unit of every connection, -1 for the others
};

// A MaxPool2dConnection's or MaxPoo3dConnection's rates, double-buffered: the gather of step t reads slot
// pool_rate_slot(T, t), where slot 0 is the caller's snn_conn_t::pool_rates and slot 1 DevNet::pool_r1, so that the last
// step's rates are the caller's.  The rates step t reads are written one slot earlier, by whoever finalises the spikes
// they fold in (pool_rate_step).
__host__ __device__ __forceinline__ bool snn_is_maxpool(int kind) { return kind == SNN_CONN_MAXPOOL2D || kind == SNN_CONN_MAXPOOL3D; }
// The connection kinds that only the POOL instantiation of the generic kernel runs (the plan selects it when one is
// present); none of them is gathered through the dense path of phase 1.
__host__ __device__ __forceinline__ bool snn_pool_inst_kind(int kind) {
    return snn_is_maxpool(kind) || kind == SNN_CONN_LOCAL2D || kind == SNN_CONN_CONV3D || kind == SNN_CONN_CONV1D ||
           kind == SNN_CONN_LOCAL3D;
}
// One axis of a pooling geometry: F.max_pool2d / F.max_pool3d's output size (no ceil mode) and padding limit (at most
// half the kernel), and at least one element inside the input in every window.
static inline bool snn_pool_axis_ok(int in, int out, int k, int s, int p, int d) {
    if (in < 1 || k < 1 || s < 1 || d < 1 || p < 0 || p > k / 2) return false;
    const int e = in + 2 * p - d * (k - 1) - 1;
    if (e < 0 || out != e / s + 1) return false;
    for (int o = 0; o < out; ++o) {
        bool any = false;
        for (int j = 0; j < k && !any; ++j) any = o * s - p + j * d >= 0 && o * s - p + j * d < in;
        if (!any) return false;
    }
    return true;
}
// A MaxPool2dConnection's or MaxPoo3dConnection's geometry (snn_b200.h): cin = cout, the layer sizes and every axis
// (snn_pool_axis_ok); the depth fields are read for SNN_CONN_MAXPOOL3D only (on SNN_CONN_MAXPOOL2D they overlay the NULL
// sparse pointers).
static inline int snn_pool_geometry_ok(const snn_conn_t &C, int n_src, int n_tgt) {
    if (!C.pool_rates) return SNN_ERR_BAD_ARG;
    const bool d3 = C.kind == SNN_CONN_MAXPOOL3D;
    const long long din = d3 ? C.din : 1, dout = d3 ? C.dout : 1;
    if (C.cin != C.cout || C.cin < 1 || (long long)C.cin * din * C.hin * C.win != n_src || (long long)C.cout * dout * C.hout * C.wout != n_tgt)
        return SNN_ERR_BAD_ARG;
    if (d3 && !snn_pool_axis_ok(C.din, C.dout, C.kd, C.sd, C.pd, C.dd)) return SNN_ERR_BAD_ARG;
    if (!snn_pool_axis_ok(C.hin, C.hout, C.kh, C.sh, C.ph, C.dh) || !snn_pool_axis_ok(C.win, C.wout, C.kw, C.sw, C.pw, C.dw))
        return SNN_ERR_BAD_ARG;
    return SNN_OK;
}

// A LocalConnection2D's geometry (snn_b200.h): the layer sizes, the reference's output size int((hin - kh) / sh) + 1 of
// a window that fits, no padding or dilation, w present and no bias.
static inline int snn_local2d_geometry_ok(const snn_conn_t &C, int n_src, int n_tgt) {
    if (!C.w || C.b) return SNN_ERR_BAD_ARG;
    if (C.cin < 1 || C.cout < 1 || C.kh < 1 || C.kw < 1 || C.sh < 1 || C.sw < 1) return SNN_ERR_BAD_ARG;
    if (C.ph != 0 || C.pw != 0 || C.dh != 1 || C.dw != 1 || C.kh > C.hin || C.kw > C.win) return SNN_ERR_BAD_ARG;
    if (C.hout != (C.hin - C.kh) / C.sh + 1 || C.wout != (C.win - C.kw) / C.sw + 1) return SNN_ERR_BAD_ARG;
    if ((long long)C.cin * C.hin * C.win != n_src || (long long)C.cout * C.hout * C.wout != n_tgt) return SNN_ERR_BAD_ARG;
    return SNN_OK;
}

// A LocalConnection3D's geometry (snn_b200.h): snn_local2d_geometry_ok on three axes, the depth axis in the fields
// SNN_CONN_CONV3D uses.
static inline int snn_local3d_geometry_ok(const snn_conn_t &C, int n_src, int n_tgt) {
    if (!C.w || C.b) return SNN_ERR_BAD_ARG;
    if (C.cin < 1 || C.cout < 1 || C.kd < 1 || C.kh < 1 || C.kw < 1 || C.sd < 1 || C.sh < 1 || C.sw < 1) return SNN_ERR_BAD_ARG;
    if (C.pd != 0 || C.ph != 0 || C.pw != 0 || C.dh != 1 || C.dw != 1) return SNN_ERR_BAD_ARG;
    if (C.kd > C.din || C.kh > C.hin || C.kw > C.win) return SNN_ERR_BAD_ARG;
    if (C.dout != (C.din - C.kd) / C.sd + 1 || C.hout != (C.hin - C.kh) / C.sh + 1 || C.wout != (C.win - C.kw) / C.sw + 1)
        return SNN_ERR_BAD_ARG;
    if ((long long)C.cin * C.din * C.hin * C.win != n_src || (long long)C.cout * C.dout * C.hout * C.wout != n_tgt) return SNN_ERR_BAD_ARG;
    return SNN_OK;
}
static inline bool snn_local_rule_ok(const snn_conn_t &C) {
    return C.rule == SNN_RULE_NONE || C.rule == SNN_RULE_NOOP || C.rule == SNN_RULE_POSTPRE || C.rule == SNN_RULE_WDEP_POSTPRE ||
           C.rule == SNN_RULE_HEBBIAN;
}

// A Conv3dConnection's geometry (snn_b200.h): the layer sizes, every output size (in - k + 2p) / s + 1 of a kernel that
// fits the padded input, no dilation, w and b present.
static inline int snn_conv3d_out(int in, int k, int s, int p) { return in + 2 * p < k ? 0 : (in - k + 2 * p) / s + 1; }
static inline int snn_conv3d_geometry_ok(const snn_conn_t &C, int n_src, int n_tgt) {
    if (!C.w || !C.b) return SNN_ERR_BAD_ARG;
    if (C.cin < 1 || C.cout < 1 || C.kd < 1 || C.kh < 1 || C.kw < 1 || C.sd < 1 || C.sh < 1 || C.sw < 1) return SNN_ERR_BAD_ARG;
    if (C.pd < 0 || C.ph < 0 || C.pw < 0 || C.dh != 1 || C.dw != 1) return SNN_ERR_BAD_ARG;
    if (C.din < 1 || C.hin < 1 || C.win < 1 || C.dout < 1 || C.hout < 1 || C.wout < 1) return SNN_ERR_BAD_ARG;
    if (C.dout != snn_conv3d_out(C.din, C.kd, C.sd, C.pd) || C.hout != snn_conv3d_out(C.hin, C.kh, C.sh, C.ph) ||
        C.wout != snn_conv3d_out(C.win, C.kw, C.sw, C.pw))
        return SNN_ERR_BAD_ARG;
    if ((long long)C.cin * C.din * C.hin * C.win != n_src || (long long)C.cout * C.dout * C.hout * C.wout != n_tgt) return SNN_ERR_BAD_ARG;
    return SNN_OK;
}
// A Conv1dConnection's geometry (snn_b200.h): the layer sizes, the output size of a kernel that fits the padded input,
// the height axis set to 1, no dilation, w and b present.
static inline int snn_conv1d_geometry_ok(const snn_conn_t &C, int n_src, int n_tgt) {
    if (!C.w || !C.b) return SNN_ERR_BAD_ARG;
    if (C.cin < 1 || C.cout < 1 || C.kw < 1 || C.sw < 1 || C.pw < 0 || C.win < 1 || C.wout < 1) return SNN_ERR_BAD_ARG;
    if (C.hin != 1 || C.hout != 1 || C.kh != 1 || C.sh != 1 || C.ph != 0 || C.dh != 1 || C.dw != 1) return SNN_ERR_BAD_ARG;
    if (C.wout != snn_conv3d_out(C.win, C.kw, C.sw, C.pw)) return SNN_ERR_BAD_ARG;
    if ((long long)C.cin * C.win != n_src || (long long)C.cout * C.wout != n_tgt) return SNN_ERR_BAD_ARG;
    return SNN_OK;
}
static inline bool snn_conv1d_rule_ok(const snn_conn_t &C) {
    return C.rule == SNN_RULE_NONE || C.rule == SNN_RULE_NOOP || C.rule == SNN_RULE_POSTPRE || C.rule == SNN_RULE_WDEP_POSTPRE ||
           C.rule == SNN_RULE_HEBBIAN;
}
// The updates a Conv3dConnection runs (snn_b200.h): none, learning.NoOp's decay, or a zero-rate PostPre /
// WeightDependentPostPre (decay and clamp).
static inline bool snn_conv3d_rule_ok(const snn_conn_t &C) {
    if (C.rule == SNN_RULE_NONE || C.rule == SNN_RULE_NOOP) return true;
    return (C.rule == SNN_RULE_POSTPRE || C.rule == SNN_RULE_WDEP_POSTPRE) && C.nu0 == 0.0f && C.nu1 == 0.0f;
}

// The per-synapse tensors of a dense connection (snn_b200.h): known forms, the rate pair set together, PostPre's rates
// broadcast to [1, n_tgt] (any other shape is the reference's bmm error), and no MCC-only rule.
static inline int snn_syn_check(const snn_conn_t &C) {
    auto form_ok = [](const float *t, int f) { return !t || (f >= SNN_SYN_FULL && f <= SNN_SYN_ONE); };
    if (!form_ok(C.wmin_t, C.wmin_form) || !form_ok(C.wmax_t, C.wmax_form) || !form_ok(C.nu0_t, C.nu0_form) || !form_ok(C.nu1_t, C.nu1_form))
        return SNN_ERR_BAD_ARG;
    if ((C.nu0_t == nullptr) != (C.nu1_t == nullptr) || C.rule == SNN_RULE_MCC_POSTPRE) return SNN_ERR_BAD_ARG;
    if (C.rule == SNN_RULE_POSTPRE && C.nu0_t && ((C.nu0_form != SNN_SYN_TGT && C.nu0_form != SNN_SYN_ONE) ||
                                                  (C.nu1_form != SNN_SYN_TGT && C.nu1_form != SNN_SYN_ONE)))
        return SNN_ERR_BAD_ARG;
    return SNN_OK;
}

__host__ __device__ __forceinline__ int pool_rate_slot(int T, int t) { return (T - 1 - t) & 1; }
__device__ __forceinline__ float *pool_rates_at(const DevNet &N, int c, int slot) { return slot ? N.pool_r1[c] : N.conns[c].pool_rates; }
// MaxPool2dConnection / MaxPoo3dConnection.compute step 1 (topology.py:1175-1176, :1265-1266): r -= decay * r; r += s
__host__ __device__ __forceinline__ float pool_rate_update(float r, float decay, bool s) {
    r = r - decay * r;
    return r + (s ? 1.0f : 0.0f);
}

__device__ __forceinline__ unsigned int ld_acquire_u32(const unsigned int *p) {
#ifdef SNN_EMU
    return __atomic_load_n(p, __ATOMIC_ACQUIRE);
#else
    unsigned int v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
#endif
}
__device__ __forceinline__ void st_release_u32(unsigned int *p, unsigned int v) {
#ifdef SNN_EMU
    __atomic_store_n(p, v, __ATOMIC_RELEASE);
#else
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
#endif
}

// Grid barrier on ONE monotonic arrival counter in global memory: a release reduction to arrive (no return value:
// one L2 transaction), relaxed polling of the same word with a short back-off until `gen * nblocks` arrivals are in,
// then one acquire fence.  `gen` is the caller's barrier count (a register, identical in every CTA).  Requires all
// CTAs of the grid to be co-resident (cooperative launch).  A time-out (~2 s) raises SNN_ERR_BARRIER and makes every
// CTA leave the time loop instead of hanging the device: the CTA that gives up adds 2^30 to the counter, which
// releases every present and future wait and is recognised as "abort" by whoever reads it.  The pollers back off
// (nanosleep): in the generic kernel many CTAs wait here while others still stream state and weights through L2.
__device__ __forceinline__ bool grid_barrier(unsigned int *bar, unsigned int nblocks, int32_t *err, unsigned int &gen) {
#ifdef SNN_EMU
    int &s_abort = emu::tls_cta->s_abort;
#else
    __shared__ int s_abort;
#endif
    ++gen;
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned int target = gen * nblocks;
#ifdef SNN_EMU
        __atomic_fetch_add(bar, 1u, __ATOMIC_RELEASE);
#else
        asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(bar) : "memory");
#endif
        int ab = 0;
        const long long t0 = clock64();
        unsigned int ns = 20;
        for (;;) {
            unsigned int v;
#ifdef SNN_EMU
            v = __atomic_load_n(bar, __ATOMIC_ACQUIRE);
#else
            asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(bar) : "memory");
#endif
            if ((int)(v - target) >= 0) { ab = (v - target) >= 0x20000000u; break; }
            __nanosleep(ns);
            if (ns < 160) ns += 20;
            if (clock64() - t0 > 4000000000LL) {
                if (err) atomicOr(err, SNN_ERR_BARRIER);
                atomicAdd(bar, 0x40000000u);
                ab = 1;
                break;
            }
        }
#ifdef SNN_EMU
        __atomic_thread_fence(__ATOMIC_SEQ_CST);
#else
        asm volatile("fence.acq_rel.gpu;" ::: "memory");
#endif
        s_abort = ab;
    }
    __syncthreads();
    return s_abort == 0;
}

__device__ __forceinline__ float clampf(float w, float lo, float hi) {
    w = w < lo ? lo : w;
    w = w > hi ? hi : w;
    return w;
}

// Nodes.forward trace update (nodes.py:96-103): decay, then set / add on spike.
__device__ __forceinline__ float trace_step(float x, bool s, float decay, float scale, int additive) {
    x = x * decay;
    if (additive) x = x + scale * (s ? 1.0f : 0.0f);
    else if (s) x = scale;
    return x;
}

// The parameters a neuron of an SNN_NODE_LIF / SNN_NODE_DC layer reads (snn_b200.h SNN_NODE_PN): the layer's scalars, or
// the neuron's row of the per-neuron block where pn_mask has the bit.
struct NeuronPar {
    float thresh, rest, decay, theta_plus, theta_decay, trace_decay, trace_scale;
};
// pn_mask of a layer whose storage holds a per-neuron block (the library zeroes it on LIF / DC layers without the flag)
__device__ __forceinline__ uint32_t pn_mask_of(const snn_layer_t &L) {
    return L.kind == SNN_NODE_LIF || L.kind == SNN_NODE_DC ? L.pn_mask : 0u;
}
__device__ __forceinline__ float pn_at(const snn_layer_t &L, uint32_t mask, int row, float scalar, int j) {
    return (mask >> row) & 1u ? __ldg(L.pn + (size_t)row * L.n + j) : scalar;
}
__device__ __forceinline__ NeuronPar neuron_par(const snn_layer_t &L, int j) {
    const uint32_t m = pn_mask_of(L);
    NeuronPar P;
    P.thresh = pn_at(L, m, SNN_PN_THRESH, L.thresh, j);
    P.rest = pn_at(L, m, SNN_PN_REST, L.rest, j);
    P.decay = pn_at(L, m, SNN_PN_DECAY, L.decay, j);
    P.theta_plus = pn_at(L, m, SNN_PN_THETA_PLUS, L.theta_plus, j);
    P.theta_decay = pn_at(L, m, SNN_PN_THETA_DECAY, L.theta_decay, j);
    P.trace_decay = pn_at(L, m, SNN_PN_TRACE_DECAY, L.trace_decay, j);
    P.trace_scale = pn_at(L, m, SNN_PN_TRACE_SCALE, L.trace_scale, j);
    return P;
}

// LIFNodes.forward (nodes.py:500-529) with the neuron's decay, rest and threshold.  `xin` is masked in place like the
// reference does.
__device__ __forceinline__ bool lif_step_p(const snn_layer_t &L, float decay, float rest, float thresh, float &v, float &rc, float &xin) {
    v = decay * (v - rest) + rest;
    if (rc > 0.0f) xin = 0.0f;
    rc = rc - L.dt;
    v = v + xin;
    const bool s = v >= thresh;
    if (s) { rc = L.refrac; v = L.reset; }
    if (L.has_lbound && v < L.lbound) v = L.lbound;
    return s;
}
__device__ __forceinline__ bool lif_step(const snn_layer_t &L, float &v, float &rc, float &xin) {
    return lif_step_p(L, L.decay, L.rest, L.thresh, v, rc, xin);
}

// IFNodes.forward (nodes.py:377-394): no leak, the gate is taken before the refractory decrement, x stays unmasked.
__device__ __forceinline__ bool if_step(const snn_layer_t &L, float &v, float &rc, float xin) {
    const float gate = rc <= 0.0f ? 1.0f : 0.0f;
    v = v + gate * xin;
    rc = rc - L.dt;
    const bool s = v >= L.thresh;
    if (s) { rc = L.refrac; v = L.reset; }
    if (L.has_lbound && v < L.lbound) v = L.lbound;
    return s;
}

// SubtractiveResetIFNodes.forward (conversion/nodes.py:73-99): the gate is rc == 0 (a negative rc, left by
// 0 < rc < dt, gates the next step's input off), the decrement keeps rc only while it is positive (else -0.0), and a
// spike subtracts the threshold instead of resetting.
__device__ __forceinline__ bool subif_step(const snn_layer_t &L, float &v, float &rc, float xin) {
    const float gate = rc == 0.0f ? 1.0f : 0.0f;
    v = v + gate * xin;
    rc = (rc > 0.0f ? 1.0f : 0.0f) * (rc - L.dt);
    const bool s = v >= L.thresh;
    if (s) { rc = L.refrac; v = v - L.thresh; }
    if (L.has_lbound && v < L.lbound) v = L.lbound;
    return s;
}

// A PassThroughNodes layer's state s (float32 0.0 / 1.0, snn_b200.h) as a spike; any other value raises
// SNN_ERR_NONBINARY.
__device__ __forceinline__ bool passthrough_spike(const snn_layer_t &L, size_t k, int32_t *err) {
    const float f = ((const float *)L.s)[k];
    if (f != 0.0f && f != 1.0f && err) atomicOr(err, SNN_ERR_NONBINARY);
    return f != 0.0f;
}

// CurrentLIFNodes.forward (nodes.py:770-791): decaying synaptic current `ic`, gate taken after the decrement.
__device__ __forceinline__ bool clif_step(const snn_layer_t &L, float &v, float &rc, float &ic, float xin) {
    v = L.decay * (v - L.rest) + L.rest;
    ic = ic * L.i_decay;
    rc = rc - L.dt;
    ic = ic + xin;
    const float gate = rc <= 0.0f ? 1.0f : 0.0f;
    v = v + gate * ic;
    const bool s = v >= L.thresh;
    if (s) { rc = L.refrac; v = L.reset; }
    if (L.has_lbound && v < L.lbound) v = L.lbound;
    return s;
}

// BoostedLIFNodes.forward (nodes.py:620-647): v *= decay, x masked in place while refractory, reset to 0.
__device__ __forceinline__ bool boosted_step(const snn_layer_t &L, float &v, float &rc, float &xin) {
    v = v * L.decay;
    if (rc > 0.0f) xin = 0.0f;
    rc = rc - L.dt;
    v = v + xin;
    const bool s = v >= L.thresh;
    if (s) { rc = L.refrac; v = 0.0f; }
    return s;
}

// DiehlAndCookNodes.forward up to the threshold test (nodes.py:1077-1092); `theta` is the
// already decayed adaptive threshold of the neuron.  Returns the candidate flag.  dc_step_p: with the neuron's decay,
// rest and threshold.
__device__ __forceinline__ bool dc_step_p(const snn_layer_t &L, float decay, float rest, float thresh, float &v, float &rc, float xin,
                                          float theta) {
    v = decay * (v - rest) + rest;
    const float gate = rc <= 0.0f ? 1.0f : 0.0f;
    v = v + gate * xin;
    rc = rc - L.dt;
    const bool s = v >= (thresh + theta);
    if (s) { rc = L.refrac; v = L.reset; }
    return s;
}
__device__ __forceinline__ bool dc_step(const snn_layer_t &L, float &v, float &rc, float xin, float theta) {
    return dc_step_p(L, L.decay, L.rest, L.thresh, v, rc, xin, theta);
}

// One STDP-family update of a single synapse, in the reference's order: pre term, post term,
// weight decay, clamp (learning.py:87-104,390-420,626-653,1110-1136; MCC_learning.py:86-110,224-302).
// U / V are the batch-reduced outer products of this step for this synapse (0 if untouched).
__device__ __forceinline__ float apply_rule(const snn_conn_t &C, float w, float U, bool pre_t, float V, bool post_t) {
    if (C.rule == SNN_RULE_WDEP_POSTPRE) {
        float upd = 0.0f;
        if (C.nu0 != 0.0f) upd = upd - (C.nu0 * (pre_t ? U : 0.0f)) * (w - C.wmin);
        if (C.nu1 != 0.0f) upd = upd + (C.nu1 * (post_t ? V : 0.0f)) * (C.wmax - w);
        w = w + upd;
    } else if (C.rule == SNN_RULE_MCC_POSTPRE) {
        if (pre_t) w = w - U * C.dt_scale;
        if (post_t) w = w + V * C.dt_scale;
    } else if (C.rule == SNN_RULE_POSTPRE) {
        if (pre_t) w = w - U;
        if (post_t) w = w + V;
    } else if (C.rule == SNN_RULE_HEBBIAN) {   // learning.py:1124-1134: U / V are the plain reduced sums
        if (C.nu0 != 0.0f) w = w + C.nu0 * (pre_t ? U : 0.0f);
        if (C.nu1 != 0.0f) w = w + C.nu1 * (post_t ? V : 0.0f);
    }
    if (C.weight_decay != 0.0f) w = w * C.weight_decay;
    if (C.has_clamp) w = clampf(w, C.wmin, C.wmax);
    return w;
}

// A dense connection's per-synapse tensors (snn_b200.h wmin_t / wmax_t / nu0_t / nu1_t).  Plans that hold one run the
// SYN instantiation of the learning phase; the others never read these fields.
__host__ __device__ inline bool snn_has_syn(const snn_conn_t &C) {
    return C.kind == SNN_CONN_DENSE && (C.wmin_t || C.wmax_t || C.nu0_t || C.nu1_t);
}
// element (i, j) of a tensor in broadcast form `form`, or the scalar when there is no tensor
__device__ __forceinline__ float syn_at(const float *t, int form, float scalar, int i, int j, int nt) {
    if (!t) return scalar;
    const size_t k = form == SNN_SYN_FULL ? (size_t)i * nt + j : form == SNN_SYN_TGT ? (size_t)j : form == SNN_SYN_SRC ? (size_t)i : 0;
    return __ldg(t + k);
}
// apply_rule with the bounds and rates of synapse (i, j).  POSTPRE's rates are inside U / V already (the staged
// fl(x_tgt * nu0[j]) and x_src * nu1[j]); HEBBIAN's gates are 1 (snn_b200.h), so its rates apply ungated like the
// reference's.
__device__ __forceinline__ float apply_rule_syn(const snn_conn_t &C, float w, float U, bool pre_t, float V, bool post_t, int i, int j,
                                                int nt) {
    if (C.rule == SNN_RULE_WDEP_POSTPRE) {
        float upd = 0.0f;
        if (C.nu0 != 0.0f) upd = upd - (syn_at(C.nu0_t, C.nu0_form, C.nu0, i, j, nt) * (pre_t ? U : 0.0f)) * (w - syn_at(C.wmin_t, C.wmin_form, C.wmin, i, j, nt));
        if (C.nu1 != 0.0f) upd = upd + (syn_at(C.nu1_t, C.nu1_form, C.nu1, i, j, nt) * (post_t ? V : 0.0f)) * (syn_at(C.wmax_t, C.wmax_form, C.wmax, i, j, nt) - w);
        w = w + upd;
    } else if (C.rule == SNN_RULE_POSTPRE) {
        if (pre_t) w = w - U;
        if (post_t) w = w + V;
    } else if (C.rule == SNN_RULE_HEBBIAN) {
        if (C.nu0 != 0.0f) w = w + syn_at(C.nu0_t, C.nu0_form, C.nu0, i, j, nt) * (pre_t ? U : 0.0f);
        if (C.nu1 != 0.0f) w = w + syn_at(C.nu1_t, C.nu1_form, C.nu1, i, j, nt) * (post_t ? V : 0.0f);
    }
    if (C.weight_decay != 0.0f) w = w * C.weight_decay;
    if (C.has_clamp) w = clampf(w, syn_at(C.wmin_t, C.wmin_form, C.wmin, i, j, nt), syn_at(C.wmax_t, C.wmax_form, C.wmax, i, j, nt));
    return w;
}

static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
