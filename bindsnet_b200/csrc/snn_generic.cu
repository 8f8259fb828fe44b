// snn_generic.cu — generic persistent window kernel (any topology of Input / McCullochPitts / IF / LIF / BoostedLIF /
// CurrentLIF / DiehlAndCook / SubtractiveResetIF / PassThrough populations joined by dense, convolutional, sparse,
// pooling, 2-D and 3-D locally connected and mean-field connections).
//
// One cooperative grid iterates the whole T-step window of Network.run (reference:
// bindsnet/network/network.py:380-465) with at most four grid barriers per step and no host involvement.
// State and weights live in global memory (L2-resident); every phase of a step is cut into work units small
// enough to fill the chip, and the units of different phases need not belong to the same CTA — what one phase
// writes the next one reads through L2 (ld.cg) after a grid barrier:
//   phase 1  unit = (layer, 32-neuron tile, sample chunk): currents from bits[rd] (network.py:211-250), neuron
//            update (nodes.py), candidates -> atomicMax keys (DC one_spike) or final spikes -> bits[wr], traces;
//            the batch sum behind theta is an integer atomic per column
//   barrier  (only if some DiehlAndCookNodes layer has one_spike)
//   phase 2  one_spike layers, same units: resolve the winner per sample, final spikes, traces
//   barrier
//   phase 3  unit = (connection, 32-column tile, chunk of source rows): STDP + decay + clamp
//            (learning.py / MCC_learning.py); dense MSTDP by source tiles; conv and local rules spread over the grid
//   barrier  (+ masks + barrier when Network.run got masks)
// With a SparseConnection (the <CTAS, true> instantiation): a window pre-pass builds the column-block tables of the
// patterns, and every step starts with the sparse gather (unit = (connection, column block, sample chunk)) and a
// barrier; in one-step mode the gather of a layer's sparse inputs precedes that layer's phase 1.
// After the last step: theta, normalize() by tiles (network.py:464-465).
#include <algorithm>
#include <cstdio>
#include <cstdlib>

#include "snn_phases.cuh"

namespace {

__device__ __forceinline__ void item_of(const DevNet &N, int item, int &li, int &tile) {
    li = 0;
    #pragma unroll 1
    for (int l = 0; l < N.n_layers; ++l)
        if (item >= N.layers[l].item0) li = l;
    tile = item - N.layers[li].item0;
}

// sparse gather unit u -> (connection, column block, sample chunk)
__device__ __forceinline__ void sparse_unit(const DevNet &N, int u, int &c, int &blk, int &chunk) {
    c = 0;
    #pragma unroll 1
    for (int cc = 0; cc < N.n_conns; ++cc)
        if (N.conns[cc].kind == SNN_CONN_SPARSE && u >= N.sp[cc].first) c = cc;
    const int v = u - N.sp[c].first;
    blk = v % N.sp[c].nb;
    chunk = v / N.sp[c].nb;
}

// CTAS = CTAs per SM the variant is compiled for: 2 (128 registers) is what runs by default — the 3-CTA variant's
// 80-register budget makes it spill; it stays selectable for experiments (SNN_B200_GVAR=3).
// SPARSE: the plan holds a SparseConnection.  Plans without one run the instantiation without the sparse phases, whose
// code (and register allocation) is exactly what it is without the feature.
// FEAT: the plan holds a MulticompartmentConnection with Probability / Mask / Intensity features (snn_b200.h); only the
// dense gather of phase 1 differs.  The two are not combined in one plan.
// POOL: the plan holds a connection of a kind snn_pool_inst_kind names (MaxPool2dConnection, MaxPoo3dConnection,
// LocalConnection2D, LocalConnection3D, Conv3dConnection, Conv1dConnection) or a layer of ann_to_snn's kinds (SNN_NODE_SUBIF, SNN_NODE_PASSTHROUGH, whose s is float32): phase 1
// gathers the pooled spikes, the 2-D and 3-D local receptive fields and the 3-D and 1-D convolutions and steps those
// layers, the learning phase runs the local and Conv1d rules and the Conv3d decay over the grid, normalize() scales the local rows and the 3-D and 1-D filters, and every
// finalised spike of a pooling source advances its rates (pool_rate_step); the prologue writes the rates of step 0.  Not
// combined with SPARSE or FEAT.  The
// barriers are those of the plain window: the rates a gather reads were written before the barrier that ends the previous
// step (or, in one-step mode, before the barrier that ends the source layer).
// SYN: some dense connection carries per-synapse bounds or rates (snn_b200.h); only the learning phase differs, and
// plans without them run the instantiation whose code never reads those fields.  Not combined with SPARSE, FEAT or POOL.
// PN: some LIF / DC layer carries per-neuron parameters (snn_b200.h SNN_NODE_PN); phases 1 and 2 and the theta of the
// last step read a lane's own values where the other instantiations read the layer's scalars.  Combined with SYN only.
// AVG: some MCC PostPre averages its updates (snn_b200.h SNN_RULE_AVG); only the learning phase (and the prologue's copy
// of the slot bitmaps) differs.  Combined with FEAT only.
// WN: some dense or MCC connection carries a per-target norm tensor or normalises every step (snn_b200.h
// SNN_CONN_WNORM).  A step-normalised Weight adds one pass after the barrier that ends phases 1 / 2 (a unit per column
// tile, as at window end) and one grid barrier behind it; its clamping rule then visits every row.  Combined with FEAT
// only.
template <int CTAS, bool SPARSE, bool FEAT, bool POOL, bool SYN = false, bool PN = false, bool AVG = false, bool WN = false>
__global__ void __launch_bounds__(SNN_GEN_THREADS, CTAS) snn_generic_window(const __grid_constant__ DevNet N) {
#ifdef SNN_EMU
    float *smem = emu::tls_cta->dyn_smem;
#else
    extern __shared__ float smem[];
#endif
    const GenSmem M = gen_carve(smem, N.B);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned int G = gridDim.x;
    const int nch = N.nch;
    unsigned int bgen = 0;   // barriers passed so far (grid_barrier)
    long long pc[8] = {0, 0, 0, 0, 0, 0, 0, 0}, pt = clock64();   // phase timers (profiling only)
    #define GPROF(k) { if (N.prof && threadIdx.x == 0) { const long long now_ = clock64(); pc[k] += now_ - pt; pt = now_; } }

    // prologue: pack the incoming spike state s(-1) into slot 1, clear the arg-max keys and the theta counters
    for (int item = blockIdx.x; item < N.total_items; item += G) {
        int li, tile; item_of(N, item, li, tile);
        const DevLayer &D = N.layers[li];
        const int j = tile * SNN_TILE + lane;
        int nsp = 0;   // (a MeanFieldConnection source) s(-1) counted into slot 2, the slot of step -1
        for (int b = warp; b < N.B; b += SNN_GEN_WARPS) {
            const size_t k = (size_t)b * D.L.n + j;
            const bool s = j < D.L.n && (POOL && D.L.kind == SNN_NODE_PASSTHROUGH ? passthrough_spike(D.L, k, N.err) : D.L.s[k] != 0);
            const uint32_t w = __ballot_sync(0xffffffffu, s);
            if (lane == 0) D.bits[((size_t)1 * N.B + b) * D.nw + tile] = w;
            nsp += __popc(w);
        }
        if (D.spc && lane == 0 && nsp) atomicAdd(D.spc + 2, nsp);
        if (D.keys && tile == 0)
            for (int b = threadIdx.x; b < 2 * N.B; b += blockDim.x) D.keys[b] = 0ull;
        if (D.thcnt && warp < 3 && j < D.L.n) D.thcnt[(size_t)warp * D.L.n + j] = 0;
        if (D.anyf && tile == 0)   // slot 2 = step -1: "may have spiked" (conservative); slots 0 / 1 start empty
            for (int b = threadIdx.x; b < 3 * N.B; b += blockDim.x) D.anyf[b] = b >= 2 * N.B ? 1u : 0u;
        // MSTDP state: step t reads slot (t + T) & 1; for an odd T the first read is slot 1, so the
        // caller's tensors (slot 0) are copied there — the last step then writes slot 0
        if (N.learning && (N.T & 1))
            for (int c = 0; c < N.n_conns; ++c) {
                const snn_conn_t &C = N.conns[c];
                if (C.tgt != li || !SNN_RULE_IS_MSTDP(C.rule)) continue;
                const DevMstdp &Ms = N.mst[c];
                const size_t ns = (size_t)N.layers[C.src].L.n, nt = (size_t)D.L.n, Bz = (size_t)N.B;
                const size_t start = (size_t)tile * SNN_GEN_THREADS + threadIdx.x, stride = (size_t)D.nw * SNN_GEN_THREADS;
                for (size_t k = start; k < Bz * ns; k += stride) { Ms.pp[1][k] = Ms.pp[0][k]; if (Ms.sp[0]) Ms.sp[1][k] = Ms.sp[0][k]; }
                for (size_t k = start; k < Bz * nt; k += stride) { Ms.pm[1][k] = Ms.pm[0][k]; if (Ms.st[0]) Ms.st[1][k] = Ms.st[0][k]; }
                if (Ms.el[0]) {
                    const size_t ne = Bz * (size_t)C.cout * C.cin * C.kh * C.kw;
                    for (size_t k = start; k < ne; k += stride) Ms.el[1][k] = Ms.el[0][k];
                }
            }
        // the slot bitmaps of an averaged MCC PostPre, by the same rule (DevAvg)
        if (AVG && N.learning && (N.T & 1) && tile == 0)
            for (int c = 0; c < N.n_conns; ++c) {
                const snn_conn_t &C = N.conns[c];
                if (C.tgt != li || !snn_is_avg(C)) continue;
                const size_t nr = (size_t)C.avg_k * N.layers[C.src].nw, nc = (size_t)C.avg_k * D.nw;
                for (size_t k = threadIdx.x; k < nr; k += SNN_GEN_THREADS) N.avg[c].rows[1][k] = N.avg[c].rows[0][k];
                for (size_t k = threadIdx.x; k < nc; k += SNN_GEN_THREADS) N.avg[c].cols[1][k] = N.avg[c].cols[0][k];
            }
        // MaxPool2d / MaxPoo3dConnection rates of step 0: the caller's rates advanced by the incoming spikes s(-1); in
        // one-step mode with the source earlier in the insertion order step 0 advances them itself, from slot
        // pool_rate_slot(T, -1)
        for (int c = 0; POOL && N.T > 0 && c < N.n_conns; ++c) {
            const snn_conn_t &C = N.conns[c];
            if (!snn_is_maxpool(C.kind) || C.src != li || j >= D.L.n) continue;
            const bool cur = N.one_step && C.src < C.tgt;
            float *dst = pool_rates_at(N, c, pool_rate_slot(N.T, cur ? -1 : 0));
            for (int b = warp; b < N.B; b += SNN_GEN_WARPS) {
                const size_t k = (size_t)b * D.L.n + j;
                const float r = C.pool_rates[k];
                const bool sp = D.L.kind == SNN_NODE_PASSTHROUGH ? ((const float *)D.L.s)[k] != 0.0f : D.L.s[k] != 0;
                dst[k] = cur ? r : pool_rate_update(r, C.pool_decay, sp);
            }
        }
    }
    for (int c = 0; SPARSE && c < N.n_conns; ++c)   // column-block tables of the SparseConnections (checks the patterns)
        if (N.conns[c].kind == SNN_CONN_SPARSE) sparse_prepass(N, c, blockIdx.x * SNN_GEN_WARPS + warp, G * SNN_GEN_WARPS);
    if (!grid_barrier(N.bar, G, N.err, bgen)) return;
    GPROF(7)

    for (int t = 0; t < N.T; ++t) {
        if (N.one_step) {
            // feed-forward mode (network.py:383-396): layer by layer in insertion order, each one reading the
            // spikes its predecessors produced in THIS step — a grid barrier per layer
            for (int l = 0; l < N.n_layers; ++l) {
                const DevLayer &D = N.layers[l];
                if (SPARSE) {   // the sparse inputs of this layer, from the spikes its phase 1 would read
                    bool any = false;
                    for (int u = blockIdx.x; u < N.sp_units; u += G) {
                        int c, blk, ch; sparse_unit(N, u, c, blk, ch);
                        if (N.conns[c].tgt == l) phase_sparse(N, c, blk, ch, N.conns[c].src < l, t, M);
                    }
                    for (int c = 0; c < N.n_conns; ++c) any |= N.conns[c].kind == SNN_CONN_SPARSE && N.conns[c].tgt == l;
                    if (any && !grid_barrier(N.bar, G, N.err, bgen)) return;
                }
                for (int u = blockIdx.x; u < D.nw * nch; u += G) phase1<SPARSE, FEAT, POOL, PN>(N, l, u / nch, u % nch, t, M);
                if (D.L.kind == SNN_NODE_DC && D.L.one_spike) {
                    if (!grid_barrier(N.bar, G, N.err, bgen)) return;
                    for (int u = blockIdx.x; u < D.nw * nch; u += G) phase2<POOL, PN>(N, l, u / nch, u % nch, t);
                }
                if (l + 1 < N.n_layers && !grid_barrier(N.bar, G, N.err, bgen)) return;
            }
        } else {
            if (SPARSE) {   // sparse inputs of step t: spikes of step t - 1, values after step t - 1's decay
                for (int u = blockIdx.x; u < N.sp_units; u += G) {
                    int c, blk, ch; sparse_unit(N, u, c, blk, ch);
                    phase_sparse(N, c, blk, ch, false, t, M);
                }
                GPROF(1)
                if (!grid_barrier(N.bar, G, N.err, bgen)) return;
                GPROF(2)
            }
            for (int u = blockIdx.x; u < N.total_items * nch; u += G) {
                int li, tile; item_of(N, u / nch, li, tile);
                phase1<SPARSE, FEAT, POOL, PN>(N, li, tile, u % nch, t, M);
            }
        }
        GPROF(0)
        if (N.any_one_spike && !N.one_step) {
            if (!grid_barrier(N.bar, G, N.err, bgen)) return;
            GPROF(1)
            for (int u = blockIdx.x; u < N.total_items * nch; u += G) {
                int li, tile; item_of(N, u / nch, li, tile);
                const snn_layer_t &L = N.layers[li].L;
                if (L.kind == SNN_NODE_DC && L.one_spike) phase2<POOL, PN>(N, li, tile, u % nch, t);
            }
            GPROF(2)
        }
        if (!grid_barrier(N.bar, G, N.err, bgen)) return;
        GPROF(3)
        if (WN && N.wn_units) {   // Weight(norm_frequency='time step'): after the step's gather, before the rule
            for (int u = blockIdx.x; u < N.wn_units; u += G) {
                int c = 0;
                #pragma unroll 1
                for (int cc = 0; cc < N.n_conns; ++cc)
                    if (N.wn_first[cc] >= 0 && u >= N.wn_first[cc]) c = cc;
                const snn_conn_t &C = N.conns[c];
                normalize_tile<true>(C, N.layers[C.src].L.n, N.layers[C.tgt].L.n, u - N.wn_first[c], M.red);
            }
            if (!grid_barrier(N.bar, G, N.err, bgen)) return;
        }
        if (N.learning) {
            for (int u = blockIdx.x; u < N.p3_total; u += G) {
                int c = 0;
                #pragma unroll 1
                for (int cc = 0; cc < N.n_conns; ++cc)
                    if (N.p3_rc[cc] > 0 && u >= N.p3_first[cc]) c = cc;
                const snn_conn_t &C = N.conns[c];
                const int v = u - N.p3_first[c];
                if (SNN_RULE_IS_MSTDP(C.rule)) {   // dense MSTDP / MSTDPET: by source tiles
                    phase3_mstdp_dense<SYN>(N, c, v, t, M);
                } else {
                    const int rcn = N.p3_rc[c], tile = v / rcn, rc = v - tile * rcn;
                    const int nwS = N.layers[C.src].nw;
                    const int wg0 = (int)((long long)rc * nwS / rcn), wg1 = (int)((long long)(rc + 1) * nwS / rcn);
                    if (AVG && snn_is_avg(C)) phase3_mcc_avg(N, c, tile, wg0, wg1, t, M);
                    else phase3<SYN, WN>(N, c, tile, wg0, wg1, t, M);
                }
            }
            GPROF(4)
            for (int c = 0; c < N.n_conns; ++c) {
                if (N.conns[c].kind == SNN_CONN_CONV2D && N.conns[c].rule != SNN_RULE_NONE) phase3_conv(N, c, blockIdx.x, G, t, M);
                if (POOL && N.conns[c].kind == SNN_CONN_LOCAL2D && N.conns[c].rule != SNN_RULE_NONE) phase3_local2d(N, c, blockIdx.x, G, t);
                if (POOL && N.conns[c].kind == SNN_CONN_CONV3D && N.conns[c].rule != SNN_RULE_NONE) phase3_conv3d(N.conns[c], blockIdx.x, G);
                if (POOL && N.conns[c].kind == SNN_CONN_CONV1D && N.conns[c].rule != SNN_RULE_NONE) phase3_conv1d(N, c, blockIdx.x, G, t);
                if (POOL && N.conns[c].kind == SNN_CONN_LOCAL3D && N.conns[c].rule != SNN_RULE_NONE) phase3_local3d(N, c, blockIdx.x, G, t);
                if (SPARSE && N.conns[c].kind == SNN_CONN_SPARSE) decay_sparse(N.conns[c], blockIdx.x, G);
            }
            GPROF(5)
            // the units of the learning phase are not the units that gather from the weights in the next step
            if (!grid_barrier(N.bar, G, N.err, bgen)) return;
            GPROF(6)
        }
        if (N.any_mask) {   // connection masks apply after the update, learning or not (topology.py:127-131)
            for (int item = blockIdx.x; item < N.total_items; item += G) {
                int li, tile; item_of(N, item, li, tile);
                for (int c = 0; c < N.n_conns; ++c) {
                    const snn_conn_t &C = N.conns[c];
                    if (C.mask && C.tgt == li && C.kind == SNN_CONN_DENSE) mask_tile(C, N.layers[C.src].L.n, N.layers[li].L.n, tile);
                }
            }
            if (!grid_barrier(N.bar, G, N.err, bgen)) return;
        }
    }

    if (N.prof && threadIdx.x == 0)
        for (int k = 0; k < 8; ++k) N.prof[blockIdx.x * 8 + k] = pc[k];
    // theta of the last step (the counters were complete at that step's barrier)
    if (N.T > 0)
        for (int item = blockIdx.x; item < N.total_items; item += G) {
            int li, tile; item_of(N, item, li, tile);
            const DevLayer &D = N.layers[li];
            const int j = tile * SNN_TILE + lane;
            if (D.thcnt && D.L.learning && warp == 0 && j < D.L.n) {
                const int tl = N.T - 1;
                const float tplus = PN ? pn_at(D.L, pn_mask_of(D.L), SNN_PN_THETA_PLUS, D.L.theta_plus, j) : D.L.theta_plus;
                D.L.theta[j] = __ldcg(D.thdec + (size_t)(tl & 1) * D.L.n + j) + tplus * (float)__ldcg(D.thcnt + (size_t)(tl % 3) * D.L.n + j);
            }
        }
    if (N.normalize) {
        for (int item = blockIdx.x; item < N.total_items; item += G) {
            int li, tile; item_of(N, item, li, tile);
            for (int c = 0; c < N.n_conns; ++c)
                if (N.conns[c].tgt == li && N.conns[c].has_norm && !(WN && N.conns[c].norm_step && N.conns[c].kind == SNN_CONN_MCC)) {
                    if (N.conns[c].kind == SNN_CONN_CONV2D) normalize_conv_item(N.conns[c], N.conns[c].kh * N.conns[c].kw, tile, N.layers[li].nw);
                    else if (POOL && N.conns[c].kind == SNN_CONN_CONV3D)
                        normalize_conv_item(N.conns[c], N.conns[c].kd * N.conns[c].kh * N.conns[c].kw, tile, N.layers[li].nw);
                    else if (POOL && N.conns[c].kind == SNN_CONN_CONV1D) normalize_conv_item(N.conns[c], N.conns[c].kw, tile, N.layers[li].nw);
                    else if (POOL && N.conns[c].kind == SNN_CONN_LOCAL2D)
                        normalize_local2d_item(N.conns[c], N.conns[c].cin * N.layers[li].L.n, N.conns[c].kh * N.conns[c].kw, tile, N.layers[li].nw);
                    else if (POOL && N.conns[c].kind == SNN_CONN_LOCAL3D)
                        normalize_local2d_item(N.conns[c], N.conns[c].cin * N.layers[li].L.n, N.conns[c].kd * N.conns[c].kh * N.conns[c].kw, tile,
                                             N.layers[li].nw);
                    else normalize_tile<WN>(N.conns[c], N.layers[N.conns[c].src].L.n, N.layers[li].L.n, tile, M.red);
                }
        }
    }
}

}  // namespace

size_t snn_generic_smem_bytes(int B) { return gen_smem_bytes(B); }

// some LIF / DC layer of the plan carries per-neuron parameters (the library keeps pn_mask zero on every other one)
static bool snn_dev_has_pn(const DevNet &N) {
    for (int l = 0; l < N.n_layers; ++l) {
        const snn_layer_t &L = N.layers[l].L;
        if ((L.kind == SNN_NODE_LIF || L.kind == SNN_NODE_DC) && L.pn_mask) return true;
    }
    return false;
}

// The work decomposition (sample chunks of phases 1 / 2, learning-phase units) for a grid of at most `cap` co-resident
// CTAs; returns the grid size.
static int plan_units(DevNet &N, int cap) {
    // phases 1 / 2: about four samples per warp and unit, but no more units than ~16 waves of the grid
    int nch = ceil_div(N.B, 4 * SNN_GEN_WARPS);
    while (nch > 1 && (long long)N.total_items * nch > 16LL * cap) --nch;
    N.cs = ceil_div(N.B, nch);
    N.nch = ceil_div(N.B, N.cs);
    // phase 3: row chunks per tile so that the units of a connection roughly fill the grid
    int p3 = 0;
    for (int c = 0; c < N.n_conns; ++c) {
        const snn_conn_t &C = N.conns[c];
        N.p3_first[c] = p3;
        N.p3_rc[c] = 0;
        if (!N.learning || C.rule == SNN_RULE_NONE || C.kind == SNN_CONN_CONV2D || C.kind == SNN_CONN_SPARSE || snn_pool_inst_kind(C.kind) ||
            C.kind == SNN_CONN_MEANFIELD)
            continue;   // (a pooling connection has no weights to update, a mean-field one's NoOp leaves them as they are;
                        // conv and local rules are spread over the grid)
        const int nwS = N.layers[C.src].nw, nwT = N.layers[C.tgt].nw;
        if (SNN_RULE_IS_MSTDP(C.rule)) { N.p3_rc[c] = 1; p3 += nwS; continue; }
        int rc = ceil_div(cap, nwT);
        const int rc_max = ceil_div(nwS, SNN_GEN_WARPS);
        if (rc > rc_max) rc = rc_max;
        if (rc < 1) rc = 1;
        N.p3_rc[c] = rc;
        p3 += nwT * rc;
    }
    N.p3_total = p3;
    // per-step normalisation: a unit per column tile of every such connection
    int wnu = 0;
    for (int c = 0; c < N.n_conns; ++c) {
        N.wn_first[c] = -1;
        if (N.conns[c].kind == SNN_CONN_MCC && N.conns[c].norm_step) { N.wn_first[c] = wnu; wnu += N.layers[N.conns[c].tgt].nw; }
    }
    N.wn_units = wnu;
    // sparse gather: (column block, chunk of SNN_GEN_WARPS samples) per SparseConnection (the blocks come from layout_generic)
    int spu = 0;
    for (int c = 0; c < N.n_conns; ++c)
        if (N.conns[c].kind == SNN_CONN_SPARSE) {
            N.sp[c].first = spu;
            spu += N.sp[c].nb * ceil_div(N.B, SNN_GEN_WARPS);
        }
    N.sp_units = spu;
    long long units = (long long)N.total_items * N.nch;
    if (p3 > units) units = p3;
    if (spu > units) units = spu;
    if (wnu > units) units = wnu;
    bool conv_rule = false;
    for (int c = 0; c < N.n_conns; ++c)
        if (N.learning && (N.conns[c].kind == SNN_CONN_CONV2D || snn_pool_inst_kind(N.conns[c].kind)) && !snn_is_maxpool(N.conns[c].kind) &&
            N.conns[c].rule != SNN_RULE_NONE)
            conv_rule = true;
    int grid = conv_rule ? cap : (int)(units < cap ? units : cap);
    return grid < 1 ? 1 : grid;
}

#ifdef SNN_EMU
// tests/emu: the kernel's CTAs run as host threads of cooperatively scheduled fibers (cuda_emu.h); a "device" of
// SNN_EMU_SMS (default 3) SMs x 2 CTAs keeps the grid small while still giving every CTA several units per phase.
int snn_generic_launch(DevNet &N, cudaStream_t) {
    int sms = 3;
    if (const char *v = getenv("SNN_EMU_SMS")) sms = atoi(v) > 0 ? atoi(v) : 3;
    const int grid = plan_units(N, sms * 2);
    if (N.any_wn && N.any_feat)
        emu::run_grid(grid, SNN_GEN_THREADS, snn_generic_smem_bytes(N.B), [](void *a) { snn_generic_window<2, false, true, false, false, false, false, true>(*(const DevNet *)a); }, &N);
    else if (N.any_wn)
        emu::run_grid(grid, SNN_GEN_THREADS, snn_generic_smem_bytes(N.B), [](void *a) { snn_generic_window<2, false, false, false, false, false, false, true>(*(const DevNet *)a); }, &N);
    else if (N.any_avg && N.any_feat)
        emu::run_grid(grid, SNN_GEN_THREADS, snn_generic_smem_bytes(N.B), [](void *a) { snn_generic_window<2, false, true, false, false, false, true>(*(const DevNet *)a); }, &N);
    else if (N.any_avg)
        emu::run_grid(grid, SNN_GEN_THREADS, snn_generic_smem_bytes(N.B), [](void *a) { snn_generic_window<2, false, false, false, false, false, true>(*(const DevNet *)a); }, &N);
    else if (N.sp_units) emu::run_grid(grid, SNN_GEN_THREADS, snn_generic_smem_bytes(N.B), [](void *a) { snn_generic_window<2, true, false, false>(*(const DevNet *)a); }, &N);
    else if (N.any_feat) emu::run_grid(grid, SNN_GEN_THREADS, snn_generic_smem_bytes(N.B), [](void *a) { snn_generic_window<2, false, true, false>(*(const DevNet *)a); }, &N);
    else if (N.any_pool) emu::run_grid(grid, SNN_GEN_THREADS, snn_generic_smem_bytes(N.B), [](void *a) { snn_generic_window<2, false, false, true>(*(const DevNet *)a); }, &N);
    else if (snn_dev_has_pn(N) && std::any_of(N.conns, N.conns + N.n_conns, snn_has_syn))
        emu::run_grid(grid, SNN_GEN_THREADS, snn_generic_smem_bytes(N.B), [](void *a) { snn_generic_window<2, false, false, false, true, true>(*(const DevNet *)a); }, &N);
    else if (snn_dev_has_pn(N))
        emu::run_grid(grid, SNN_GEN_THREADS, snn_generic_smem_bytes(N.B), [](void *a) { snn_generic_window<2, false, false, false, false, true>(*(const DevNet *)a); }, &N);
    else if (std::any_of(N.conns, N.conns + N.n_conns, snn_has_syn))
        emu::run_grid(grid, SNN_GEN_THREADS, snn_generic_smem_bytes(N.B), [](void *a) { snn_generic_window<2, false, false, false, true>(*(const DevNet *)a); }, &N);
    else emu::run_grid(grid, SNN_GEN_THREADS, snn_generic_smem_bytes(N.B), [](void *a) { snn_generic_window<2, false, false, false>(*(const DevNet *)a); }, &N);
    return 0;
}
#else
// Launch the generic window: fills in the work decomposition (sample chunks, learning-phase units) for the grid
// the device can keep co-resident.  Returns a cudaError_t cast to int.
int snn_generic_launch(DevNet &N, cudaStream_t stream) {
    int dev = 0, sms = 0, per_sm = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return (int)e;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const size_t smem = snn_generic_smem_bytes(N.B);
    // two CTAs per SM unless SNN_B200_GVAR=3 asks for the spilling three-CTA experiment (plans without a SparseConnection,
    // MCC features or the POOL instantiation's kinds)
    const bool sparse = std::any_of(N.conns, N.conns + N.n_conns, [](const snn_conn_t &C) { return C.kind == SNN_CONN_SPARSE; });
    const bool syn = std::any_of(N.conns, N.conns + N.n_conns, snn_has_syn);
    const bool pn = snn_dev_has_pn(N);
    bool three = false;
    if (const char *v = getenv("SNN_B200_GVAR"))
        three = !sparse && !N.any_feat && !N.any_pool && !syn && !pn && !N.any_avg && !N.any_wn && v[0] == '3' && 3 * (smem + 1024) <= 227 * 1024;
    const void *kern = N.any_wn ? (N.any_feat ? (const void *)snn_generic_window<2, false, true, false, false, false, false, true>
                                              : (const void *)snn_generic_window<2, false, false, false, false, false, false, true>)
                     : N.any_avg ? (N.any_feat ? (const void *)snn_generic_window<2, false, true, false, false, false, true>
                                               : (const void *)snn_generic_window<2, false, false, false, false, false, true>)
                     : three ? (const void *)snn_generic_window<3, false, false, false>
                     : sparse ? (const void *)snn_generic_window<2, true, false, false>
                     : pn ? (syn ? (const void *)snn_generic_window<2, false, false, false, true, true>
                               : (const void *)snn_generic_window<2, false, false, false, false, true>)
                     : syn ? (const void *)snn_generic_window<2, false, false, false, true>
                     : N.any_feat ? (const void *)snn_generic_window<2, false, true, false>
                     : N.any_pool ? (const void *)snn_generic_window<2, false, false, true> : (const void *)snn_generic_window<2, false, false, false>;
    e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, SNN_GEN_THREADS, smem);
    if (e != cudaSuccess) return (int)e;
    if (per_sm < 1) return (int)cudaErrorLaunchOutOfResources;
    if (per_sm > (three ? 3 : 2)) per_sm = three ? 3 : 2;
    const int grid = plan_units(N, sms * per_sm);
    static long long *prof_buf = nullptr;   // debug only (env SNN_B200_GPROF): per-phase cycles of thread 0 of every CTA
    const bool prof = getenv("SNN_B200_GPROF") != nullptr;
    if (prof) {
        if (!prof_buf && cudaMalloc(&prof_buf, sizeof(long long) * 8 * 4096) != cudaSuccess) return (int)cudaErrorMemoryAllocation;
        cudaMemsetAsync(prof_buf, 0, sizeof(long long) * 8 * 4096, stream);
        N.prof = prof_buf;
    }
    void *args[] = {(void *)&N};
    const int rc = (int)cudaLaunchCooperativeKernel(kern, dim3(grid), dim3(SNN_GEN_THREADS), args, smem, stream);
    if (prof && rc == 0 && N.T > 0) {
        static long long host[8 * 4096];
        cudaStreamSynchronize(stream);
        cudaMemcpy(host, prof_buf, sizeof(long long) * 8 * grid, cudaMemcpyDeviceToHost);
        const char *names[8] = {"phase1", "barrierA", "phase2", "barrierB", "phase3", "phase3conv", "barrierC", "prologue"};
        if (N.sp_units) { names[1] = "sparse/bA"; names[2] = "sp.bar/ph2"; }   // with a SparseConnection: + gather, + its barrier
        fprintf(stderr, "[snn_b200 gprof] grid=%d x %d threads, nch=%d cs=%d p3_units=%d T=%d B=%d  (cycles per timestep: min / mean / max over CTAs)\n",
                grid, SNN_GEN_THREADS, N.nch, N.cs, N.p3_total, N.T, N.B);
        for (int k = 0; k < 8; ++k) {
            long long mn = host[k], mx = host[k]; double sum = 0;
            for (int g = 0; g < grid; ++g) { const long long v = host[g * 8 + k]; mn = v < mn ? v : mn; mx = v > mx ? v : mx; sum += (double)v; }
            const double d = k == 7 ? 1.0 : (double)N.T;
            fprintf(stderr, "[snn_b200 gprof]   %-10s %10.0f %10.0f %10.0f\n", names[k], mn / d, sum / grid / d, mx / d);
        }
    }
    return rc;
}
#endif
