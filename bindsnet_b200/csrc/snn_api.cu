// snn_api.cu — the C ABI of libsnn_b200.so (include/snn_b200.h): plan validation, workspace
// layout, tier selection and launches.  No torch types, no host synchronisation.
#include <cstdio>
#include <cstring>

#include "snn_common.cuh"

int snn_generic_launch(DevNet &N, cudaStream_t stream);
int snn_fused_dc_supported(const snn_net_t *net, const snn_run_opts_t *opts);
size_t snn_fused_dc_workspace_bytes(const snn_net_t *net, const snn_run_opts_t *opts);
int snn_fused_dc_launch(const snn_net_t *net, const snn_run_opts_t *opts, void *ws, size_t ws_bytes,
                        cudaStream_t stream, int *launches);
int snn_fused_dc2_supported(const snn_net_t *net, const snn_run_opts_t *opts);
size_t snn_fused_dc2_workspace_bytes(const snn_net_t *net, const snn_run_opts_t *opts);
int snn_fused_dc2_launch(const snn_net_t *net, const snn_run_opts_t *opts, void *ws, size_t ws_bytes,
                         cudaStream_t stream, int *launches);

static thread_local int g_last_launches = 0;

static inline size_t align_up(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }

// A LIF / DC layer's per-neuron block (snn_b200.h SNN_NODE_PN): a flag on those kinds only, a block wherever a row is
// used, and rows only for the parameters the layer reads.
static int pn_check(const snn_layer_t &L) {
    const int kind = L.kind & ~SNN_NODE_PN;
    if (kind != SNN_NODE_LIF && kind != SNN_NODE_DC) return SNN_ERR_BAD_ARG;
    uint32_t allowed = 1u << SNN_PN_THRESH | 1u << SNN_PN_REST | 1u << SNN_PN_DECAY;
    if (kind == SNN_NODE_DC) allowed |= 1u << SNN_PN_THETA_PLUS | 1u << SNN_PN_THETA_DECAY;
    if (L.traces) allowed |= 1u << SNN_PN_TRACE_DECAY;
    if (L.traces && L.traces_additive) allowed |= 1u << SNN_PN_TRACE_SCALE;
    if ((L.pn_mask & ~allowed) || (L.pn_mask && !L.pn)) return SNN_ERR_BAD_ARG;
    return SNN_OK;
}

// An averaged MCC PostPre (snn_b200.h SNN_RULE_AVG): the rule and kind it extends, its state, no mask.
static int avg_check(const snn_conn_t &C) {
    if ((C.rule & ~SNN_RULE_AVG) != SNN_RULE_MCC_POSTPRE || C.kind != SNN_CONN_MCC || C.mask) return SNN_ERR_UNSUPPORTED;
    if (C.avg_k < 1 || C.avg_idx_pre < 0 || C.avg_idx_pre >= C.avg_k || C.avg_idx_post < 0 || C.avg_idx_post >= C.avg_k)
        return SNN_ERR_BAD_ARG;
    if (!C.avg_pre || !C.avg_post || !C.avg_rows || !C.avg_cols) return SNN_ERR_BAD_ARG;
    return SNN_OK;
}

// A dense or MCC connection's norm tensor / per-step normalisation (snn_b200.h SNN_CONN_WNORM): the kinds that have it,
// a norm to apply, a per-step flag on an MCC Weight only, and no averaged rule.
static int wnorm_check(const snn_conn_t &C) {
    const int kind = C.kind & ~SNN_CONN_WNORM;
    if (kind != SNN_CONN_DENSE && kind != SNN_CONN_MCC) return SNN_ERR_UNSUPPORTED;
    if (!C.has_norm || (C.norm_step != 0 && C.norm_step != 1)) return SNN_ERR_BAD_ARG;
    if ((C.norm_step && kind != SNN_CONN_MCC) || (C.rule & SNN_RULE_AVG)) return SNN_ERR_UNSUPPORTED;
    return SNN_OK;
}

// The plan every check and kernel below reads: the kinds without SNN_NODE_PN, pn_mask cleared on the LIF / DC layers
// that do not carry the flag (their storage is CurrentLIFNodes' otherwise); the rules without SNN_RULE_AVG, avg_k
// cleared on every other MCC PostPre (snn_is_avg); the kinds without SNN_CONN_WNORM, norm_t / norm_step cleared on every
// other dense or MCC connection.  *pn: some layer uses a per-neuron row.
static int strip_pn(const snn_net_t *net, snn_net_t *out, bool *pn) {
    *pn = false;
    if (!net || net->n_layers < 0 || net->n_layers > SNN_MAX_LAYERS) return SNN_ERR_BAD_ARG;
    if (net->n_conns < 0 || net->n_conns > SNN_MAX_CONNS) return SNN_ERR_BAD_ARG;
    *out = *net;
    for (int c = 0; c < net->n_conns; ++c) {
        snn_conn_t &C = out->conns[c];
        if (C.kind & SNN_CONN_WNORM) {
            const int rc = wnorm_check(C);
            if (rc != SNN_OK) return rc;
            C.kind &= ~SNN_CONN_WNORM;
        } else if (C.kind == SNN_CONN_DENSE || C.kind == SNN_CONN_MCC) {
            C.norm_t = nullptr;
            C.norm_step = 0;
        }
        if (C.rule & SNN_RULE_AVG) {
            const int rc = avg_check(C);
            if (rc != SNN_OK) return rc;
            C.rule &= ~SNN_RULE_AVG;
        } else if (C.rule == SNN_RULE_MCC_POSTPRE) {
            C.avg_k = 0;
        }
    }
    for (int l = 0; l < net->n_layers; ++l) {
        snn_layer_t &L = out->layers[l];
        if (L.kind & SNN_NODE_PN) {
            const int rc = pn_check(L);
            if (rc != SNN_OK) return rc;
            L.kind &= ~SNN_NODE_PN;
            *pn |= L.pn_mask != 0u;
        } else if (L.kind == SNN_NODE_LIF || L.kind == SNN_NODE_DC) {
            L.pn = nullptr;
            L.pn_mask = 0u;
        }
    }
    return SNN_OK;
}

static int validate(const snn_net_t *net, const snn_run_opts_t *o) {
    if (!net || !o || net->abi_version != SNN_ABI_VERSION) return SNN_ERR_BAD_ARG;
    if (net->n_layers < 1 || net->n_layers > SNN_MAX_LAYERS) return SNN_ERR_BAD_ARG;
    if (net->n_conns < 0 || net->n_conns > SNN_MAX_CONNS) return SNN_ERR_BAD_ARG;
    if (o->T < 0 || o->B <= 0) return SNN_ERR_BAD_ARG;
    for (int l = 0; l < net->n_layers; ++l) {
        const snn_layer_t &L = net->layers[l];
        if (L.kind < SNN_NODE_INPUT || L.kind > SNN_NODE_PASSTHROUGH) return SNN_ERR_UNSUPPORTED;
        if (L.kind == SNN_NODE_CURRENT_LIF && !L.i) return SNN_ERR_BAD_ARG;
        if (L.n <= 0 || !L.s) return SNN_ERR_BAD_ARG;
        const bool stateless = L.kind == SNN_NODE_INPUT || L.kind == SNN_NODE_PASSTHROUGH;
        if (!stateless && (!L.v || (!L.refrac_count && L.kind != SNN_NODE_MCP))) return SNN_ERR_BAD_ARG;
        if (L.kind == SNN_NODE_DC && !L.theta) return SNN_ERR_BAD_ARG;
        if (L.traces && !L.x) return SNN_ERR_BAD_ARG;
        if (L.sum_input && !L.summed) return SNN_ERR_BAD_ARG;
        if (L.ext && L.ext_dtype != SNN_EXT_U8 && L.ext_dtype != SNN_EXT_F32) return SNN_ERR_BAD_ARG;
    }
    if ((o->delta_w || o->delta_theta) && (o->normalize || !net->learning || o->one_step)) return SNN_ERR_UNSUPPORTED;
    for (int c = 0; c < net->n_conns; ++c) {
        const snn_conn_t &C = net->conns[c];
        const bool sparse = C.kind == SNN_CONN_SPARSE, pool = snn_is_maxpool(C.kind), local = C.kind == SNN_CONN_LOCAL2D;
        const bool conv3d = C.kind == SNN_CONN_CONV3D, conv1d = C.kind == SNN_CONN_CONV1D, local3d = C.kind == SNN_CONN_LOCAL3D;
        if (C.src < 0 || C.src >= net->n_layers || C.tgt < 0 || C.tgt >= net->n_layers) return SNN_ERR_BAD_ARG;
        if (pool ? (C.w || C.b) : (!C.w && !(sparse && C.nnz == 0))) return SNN_ERR_BAD_ARG;
        if (net->layers[C.tgt].kind == SNN_NODE_INPUT) return SNN_ERR_UNSUPPORTED;
        if (C.rule < SNN_RULE_NONE || C.rule > SNN_RULE_MSTDPET) return SNN_ERR_UNSUPPORTED;
        if (C.kind < SNN_CONN_DENSE || C.kind > SNN_CONN_MEANFIELD) return SNN_ERR_UNSUPPORTED;
        if (C.kind == SNN_CONN_MEANFIELD) {   // w is only read; the mean is exact below 2^24 spikes (snn_b200.h)
            if (!C.mf_off || C.b || C.mf_stride < 0 || (long long)o->B * net->layers[C.src].n >= (1LL << 24)) return SNN_ERR_BAD_ARG;
            if ((C.rule != SNN_RULE_NONE && C.rule != SNN_RULE_NOOP) || C.has_norm || C.mask) return SNN_ERR_UNSUPPORTED;
        }
        if (conv1d) {   // NoOp and the three unsupervised rules, no mask (snn_b200.h)
            const int rc = snn_conv1d_geometry_ok(C, net->layers[C.src].n, net->layers[C.tgt].n);
            if (rc != SNN_OK) return rc;
            if (!snn_conv1d_rule_ok(C) || C.mask) return SNN_ERR_UNSUPPORTED;
        }
        if (pool) {   // no weights: learning.NoOp only, nothing to normalize or mask (snn_b200.h)
            if (C.rule != SNN_RULE_NOOP || C.has_norm || C.mask) return SNN_ERR_UNSUPPORTED;
            const int rc = snn_pool_geometry_ok(C, net->layers[C.src].n, net->layers[C.tgt].n);
            if (rc != SNN_OK) return rc;
        }
        if (local) {   // per-target receptive-field weights: NoOp and the three unsupervised rules, no mask (snn_b200.h)
            const int rc = snn_local2d_geometry_ok(C, net->layers[C.src].n, net->layers[C.tgt].n);
            if (rc != SNN_OK) return rc;
            if (C.rule != SNN_RULE_NONE && C.rule != SNN_RULE_NOOP && C.rule != SNN_RULE_POSTPRE && C.rule != SNN_RULE_WDEP_POSTPRE &&
                C.rule != SNN_RULE_HEBBIAN)
                return SNN_ERR_UNSUPPORTED;
        }
        if (local3d) {   // as a LocalConnection2D, on three axes (snn_b200.h)
            const int rc = snn_local3d_geometry_ok(C, net->layers[C.src].n, net->layers[C.tgt].n);
            if (rc != SNN_OK) return rc;
            if (!snn_local_rule_ok(C) || C.mask) return SNN_ERR_UNSUPPORTED;
        }
        if (conv3d) {   // decay / clamp updates only, no mask (snn_b200.h)
            const int rc = snn_conv3d_geometry_ok(C, net->layers[C.src].n, net->layers[C.tgt].n);
            if (rc != SNN_OK) return rc;
            if ((net->learning && !snn_conv3d_rule_ok(C)) || C.mask) return SNN_ERR_UNSUPPORTED;
        }
        if (sparse) {   // a fixed pattern: static or NoOp-decayed values, no normalize, no mask (snn_b200.h)
            if (C.rule != SNN_RULE_NONE && C.rule != SNN_RULE_NOOP) return SNN_ERR_UNSUPPORTED;
            if (C.has_norm || C.mask) return SNN_ERR_UNSUPPORTED;
            if (C.nnz < 0 || !C.sp_rowptr || (C.nnz > 0 && !C.sp_col)) return SNN_ERR_BAD_ARG;
        }
        if (C.kind == SNN_CONN_CONV2D) {
            const snn_layer_t &S = net->layers[C.src], &G = net->layers[C.tgt];
            if (C.cin * C.hin * C.win != S.n || C.cout * C.hout * C.wout != G.n || !C.b) return SNN_ERR_BAD_ARG;
            if (C.kh < 1 || C.kw < 1 || C.sh < 1 || C.sw < 1 || C.dh < 1 || C.dw < 1) return SNN_ERR_BAD_ARG;
            if (C.rule == SNN_RULE_MCC_POSTPRE) return SNN_ERR_UNSUPPORTED;
            if (SNN_RULE_IS_STDP(C.rule) && (C.dh != 1 || C.dw != 1)) return SNN_ERR_UNSUPPORTED;   // im2col_indices ignores dilation
        }
        // dense or MCC Weight, batch size 1 (learning.py:2187-2249, MCC_learning.py:652-733)
        if (C.rule == SNN_RULE_MSTDPET) {
            if ((C.kind != SNN_CONN_DENSE && C.kind != SNN_CONN_MCC) || o->B != 1) return SNN_ERR_UNSUPPORTED;
            if (!C.p_plus || !C.p_minus || !C.mst_spre || !C.mst_spost || !C.e_trace) return SNN_ERR_BAD_ARG;
        }
        if (C.rule == SNN_RULE_MSTDP) {
            if (!C.p_plus || !C.p_minus) return SNN_ERR_BAD_ARG;
            if (C.kind == SNN_CONN_CONV2D) { if (!C.elig || C.dh != 1 || C.dw != 1) return SNN_ERR_BAD_ARG; }
            else if (C.kind == SNN_CONN_DENSE || C.kind == SNN_CONN_MCC) { if (!C.mst_spre || !C.mst_spost) return SNN_ERR_BAD_ARG; }
            else return SNN_ERR_UNSUPPORTED;
        }
        if (SNN_RULE_IS_STDP(C.rule) && (!net->layers[C.src].traces || !net->layers[C.tgt].traces))
            return SNN_ERR_BAD_ARG;
        if (C.mask && (C.kind != SNN_CONN_DENSE || SNN_RULE_IS_MSTDP(C.rule))) return SNN_ERR_UNSUPPORTED;
        // the feature storage holds a dense connection's per-synapse tensors (snn_b200.h); any other kind leaves it empty
        if ((C.f_prob || C.f_mask || C.f_int) && C.kind != SNN_CONN_MCC && C.kind != SNN_CONN_DENSE) return SNN_ERR_BAD_ARG;
        if (snn_has_syn(C)) {
            const int rc = snn_syn_check(C);
            if (rc != SNN_OK) return rc;
        }
        // a PassThroughNodes layer carries 0 / 1 spikes: pooled ones in, none of a rule's traces (snn_b200.h)
        const bool pass_src = net->layers[C.src].kind == SNN_NODE_PASSTHROUGH, pass_tgt = net->layers[C.tgt].kind == SNN_NODE_PASSTHROUGH;
        if (pass_tgt && C.kind != SNN_CONN_MAXPOOL2D) return SNN_ERR_UNSUPPORTED;
        if ((pass_src || pass_tgt) && C.rule != SNN_RULE_NONE && C.rule != SNN_RULE_NOOP) return SNN_ERR_UNSUPPORTED;
    }
    return SNN_OK;
}

// the plan runs the pooling instantiation of the generic kernel: a connection of a kind snn_pool_inst_kind names, or a
// layer of ann_to_snn's kinds
static bool has_pool(const snn_net_t *net) {
    for (int c = 0; c < net->n_conns; ++c)
        if (snn_pool_inst_kind(net->conns[c].kind)) return true;
    for (int l = 0; l < net->n_layers; ++l)
        if (net->layers[l].kind == SNN_NODE_SUBIF || net->layers[l].kind == SNN_NODE_PASSTHROUGH) return true;
    return false;
}

// some connection is a MeanFieldConnection: every generic instantiation runs it, the fused kernels do not
static bool has_meanfield(const snn_net_t *net) {
    for (int c = 0; c < net->n_conns; ++c)
        if (net->conns[c].kind == SNN_CONN_MEANFIELD) return true;
    return false;
}

static bool has_sparse(const snn_net_t *net) {
    for (int c = 0; c < net->n_conns; ++c)
        if (net->conns[c].kind == SNN_CONN_SPARSE) return true;
    return false;
}

// some MulticompartmentConnection carries Probability / Mask / Intensity features
static bool has_feat(const snn_net_t *net) {
    for (int c = 0; c < net->n_conns; ++c) {
        const snn_conn_t &C = net->conns[c];
        if (C.kind == SNN_CONN_MCC && (C.f_prob || C.f_mask || C.f_int)) return true;
    }
    return false;
}

// some MCC PostPre averages its updates (snn_b200.h SNN_RULE_AVG)
static bool has_avg(const snn_net_t *net) {
    for (int c = 0; c < net->n_conns; ++c)
        if (snn_is_avg(net->conns[c])) return true;
    return false;
}

// some dense or MCC connection carries a norm tensor or normalises every step (SNN_CONN_WNORM, stripped by strip_pn)
static bool has_wn(const snn_net_t *net) {
    for (int c = 0; c < net->n_conns; ++c) {
        const snn_conn_t &C = net->conns[c];
        if ((C.kind == SNN_CONN_DENSE || C.kind == SNN_CONN_MCC) && (C.norm_t || C.norm_step)) return true;
    }
    return false;
}

// some dense connection carries per-synapse bounds or rates (snn_b200.h)
static bool has_syn(const snn_net_t *net) {
    for (int c = 0; c < net->n_conns; ++c)
        if (snn_has_syn(net->conns[c])) return true;
    return false;
}

static bool layer_needs_xpub(const snn_net_t *net, int l) {
    for (int c = 0; c < net->n_conns; ++c)
        if (net->conns[c].src == l && SNN_RULE_IS_STDP(net->conns[c].rule) && net->conns[c].kind != SNN_CONN_CONV2D &&
            !snn_pool_inst_kind(net->conns[c].kind))
            return true;
    return false;
}

// Carves the generic tier's workspace; with ws == nullptr only sizes it.
static size_t layout_generic(const snn_net_t *net, const snn_run_opts_t *o, char *ws, DevNet *N) {
    size_t off = 0;
    const size_t B = (size_t)o->B;
    // the barrier counters, then the spike-count slots of the MeanFieldConnection sources (layer l: words
    // SNN_BAR_WORDS + 3 l ..., on a cache line of their own); the launch zeroes both
    if (N) N->bar = (unsigned int *)(ws + off);
    off += align_up(sizeof(unsigned int) * SNN_BAR_ZERO_WORDS);
    int items = 0;
    for (int l = 0; l < net->n_layers; ++l) {
        const snn_layer_t &L = net->layers[l];
        const int nw = (L.n + 31) / 32;
        if (N) { N->layers[l].L = L; N->layers[l].nw = nw; N->layers[l].item0 = items; }
        items += nw;
        if (N) N->layers[l].bits = (uint32_t *)(ws + off);
        off += align_up(sizeof(uint32_t) * 2 * B * nw);
        const bool os = L.kind == SNN_NODE_DC && L.one_spike;
        if (N) N->layers[l].candbits = os ? (uint32_t *)(ws + off) : nullptr;
        if (os) off += align_up(sizeof(uint32_t) * B * nw);
        if (N) N->layers[l].keys = os ? (unsigned long long *)(ws + off) : nullptr;
        if (os) off += align_up(sizeof(unsigned long long) * 2 * B);
        const bool xp = L.traces && layer_needs_xpub(net, l);
        if (N) N->layers[l].xpub = xp ? (float *)(ws + off) : nullptr;
        if (xp) off += align_up(sizeof(float) * 2 * B * L.n);
        const bool th = L.kind == SNN_NODE_DC;   // adaptive threshold: decayed value per step parity + batch counters
        if (N) N->layers[l].thdec = th ? (float *)(ws + off) : nullptr;
        if (th) off += align_up(sizeof(float) * 2 * L.n);
        if (N) N->layers[l].thcnt = th ? (int32_t *)(ws + off) : nullptr;
        if (th) off += align_up(sizeof(int32_t) * 3 * L.n);
        bool wide_src = false;   // source of a dense connection with more than one gather block
        for (int c = 0; c < net->n_conns; ++c)
            if (net->conns[c].src == l && net->conns[c].kind != SNN_CONN_CONV2D && net->conns[c].kind != SNN_CONN_MEANFIELD &&
                !snn_pool_inst_kind(net->conns[c].kind) && nw > 32)
                wide_src = true;
        bool mf_src = false;
        for (int c = 0; c < net->n_conns; ++c) mf_src |= net->conns[c].src == l && net->conns[c].kind == SNN_CONN_MEANFIELD;
        if (N) N->layers[l].spc = mf_src ? (int32_t *)(N->bar + SNN_BAR_WORDS + 3 * l) : nullptr;
        if (N) N->layers[l].anyf = wide_src ? (uint32_t *)(ws + off) : nullptr;
        if (wide_src) off += align_up(sizeof(uint32_t) * 3 * B);
        if (N && os) N->any_one_spike = 1;
    }
    if (N) N->total_items = items;
    // second slot of every MSTDP rule's state (DevMstdp)
    for (int c = 0; c < net->n_conns; ++c) {
        const snn_conn_t &C = net->conns[c];
        if (!SNN_RULE_IS_MSTDP(C.rule)) continue;
        const size_t ns = (size_t)net->layers[C.src].n, nt = (size_t)net->layers[C.tgt].n;
        auto take = [&](size_t bytes) { char *p = ws ? ws + off : nullptr; off += align_up(bytes); return p; };
        char *pp = take(sizeof(float) * B * ns), *pm = take(sizeof(float) * B * nt);
        if (N) {
            DevMstdp &M = N->mst[c];
            M.pp[0] = C.p_plus; M.pm[0] = C.p_minus; M.pp[1] = (float *)pp; M.pm[1] = (float *)pm;
        }
        if (C.kind == SNN_CONN_CONV2D) {
            char *el = take(sizeof(float) * B * (size_t)C.cout * C.cin * C.kh * C.kw);
            if (N) { N->mst[c].el[0] = C.elig; N->mst[c].el[1] = (float *)el; }
        } else {
            char *sp = take(B * ns), *st = take(B * nt);
            if (N) { N->mst[c].sp[0] = C.mst_spre; N->mst[c].st[0] = C.mst_spost; N->mst[c].sp[1] = (uint8_t *)sp; N->mst[c].st[1] = (uint8_t *)st; }
        }
    }
    // SparseConnections: the column-block offset table of the pattern and the gathered input of the current step
    for (int c = 0; c < net->n_conns; ++c) {
        const snn_conn_t &C = net->conns[c];
        if (C.kind != SNN_CONN_SPARSE) continue;
        const size_t ns = (size_t)net->layers[C.src].n, nt = (size_t)net->layers[C.tgt].n;
        const int bw = sparse_block_width((int)ns, (int)nt, o->B, C.nnz), nb = ((int)nt + bw - 1) / bw;
        if (N) { N->sp[c].bw = bw; N->sp[c].nb = nb; N->sp[c].off = (int32_t *)(ws + off); }
        off += align_up(sizeof(int32_t) * ns * (size_t)(nb + 1));
        if (N) N->sp[c].out = (float *)(ws + off);
        off += align_up(sizeof(float) * B * nt);
    }
    // averaged MCC PostPre: the second slot of the slot bitmaps (DevAvg)
    for (int c = 0; c < net->n_conns; ++c) {
        const snn_conn_t &C = net->conns[c];
        if (!snn_is_avg(C)) continue;
        const size_t nr = (size_t)C.avg_k * ((net->layers[C.src].n + 31) / 32), nc = (size_t)C.avg_k * ((net->layers[C.tgt].n + 31) / 32);
        if (N) { N->avg[c].rows[0] = C.avg_rows; N->avg[c].cols[0] = C.avg_cols; N->avg[c].rows[1] = (uint32_t *)(ws + off); }
        off += align_up(sizeof(uint32_t) * nr);
        if (N) N->avg[c].cols[1] = (uint32_t *)(ws + off);
        off += align_up(sizeof(uint32_t) * nc);
    }
    // MaxPool2d / MaxPoo3dConnections: the second slot of the rates (pool_rate_slot)
    for (int c = 0; c < net->n_conns; ++c) {
        if (!snn_is_maxpool(net->conns[c].kind)) continue;
        if (N) N->pool_r1[c] = (float *)(ws + off);
        off += align_up(sizeof(float) * B * (size_t)net->layers[net->conns[c].src].n);
    }
    return off;
}

extern "C" {

int snn_b200_abi_version(void) { return SNN_ABI_VERSION; }

const char *snn_b200_build_info(void) {
    return "libsnn_b200 sm_90a (generic window + fused DC2015 windows v1/v2), ABI " "13" ", built " __DATE__ " " __TIME__;
}

int snn_b200_last_launch_count(void) { return g_last_launches; }

// (net: the plan strip_pn left; pn: some layer carries per-neuron parameters)
static int select_tier(const snn_net_t *net, const snn_run_opts_t *opts, bool pn) {
    if (validate(net, opts) != SNN_OK) return 0;
    // one extra instantiation of the generic kernel each for sparse, feature and pooling plans (pooling: every kind
    // snn_pool_inst_kind names, and SubtractiveResetIFNodes or PassThroughNodes), not combinations (and one for plans
    // with per-synapse bounds or rates)
    if ((int)has_sparse(net) + (int)has_feat(net) + (int)has_pool(net) + (int)has_syn(net) > 1) return 0;
    // norm tensors / per-step normalisation: two more instantiations, alone or with features; generic tier only
    if (has_wn(net)) {
        if (pn || has_sparse(net) || has_pool(net) || has_syn(net) || has_avg(net)) return 0;
        return (opts->tier == 0 || opts->tier == 1) && !opts->delta_w && !opts->delta_theta ? 1 : 0;
    }
    // averaged MCC PostPre: two more instantiations, alone or with features; generic tier only
    if (has_avg(net)) {
        if (pn || has_sparse(net) || has_pool(net) || has_syn(net)) return 0;
        return (opts->tier == 0 || opts->tier == 1) && !opts->delta_w && !opts->delta_theta ? 1 : 0;
    }
    // per-neuron parameters: two more instantiations, alone or with per-synapse tensors; the fused kernels read scalars
    if (pn) {
        if (has_sparse(net) || has_feat(net) || has_pool(net)) return 0;
        return (opts->tier == 0 || opts->tier == 1) && !opts->delta_w && !opts->delta_theta ? 1 : 0;
    }
    // the fused DiehlAndCook2015 kernels (and so the delta windows) have neither the sparse, the feature, the pooling
    // nor the mean-field gather, and read scalar bounds and rates only
    if (has_sparse(net) || has_feat(net) || has_pool(net) || has_syn(net) || has_meanfield(net))
        return (opts->tier == 0 || opts->tier == 1) && !opts->delta_w && !opts->delta_theta ? 1 : 0;
    if (opts->delta_w || opts->delta_theta)   // delta windows exist in the barrier kernel only
        return (opts->tier == 0 || opts->tier == 2) && snn_fused_dc_supported(net, opts) ? 2 : 0;
    if (opts->tier == 1) return 1;
    if (opts->tier == 3) return snn_fused_dc2_supported(net, opts) ? 3 : 0;
    // auto: the barrier kernel (tier 2) wherever it applies (DESIGN.md section 4 compares the two fused kernels);
    // the column-group kernel (tier 3) takes the shapes only it matches
    if (snn_fused_dc_supported(net, opts)) return 2;
    if (opts->tier == 2) return 0;
    if (snn_fused_dc2_supported(net, opts)) return 3;
    return 1;
}

int snn_b200_select_tier(const snn_net_t *net, const snn_run_opts_t *opts) {
    snn_net_t P;
    bool pn;
    if (strip_pn(net, &P, &pn) != SNN_OK) return 0;
    return select_tier(&P, opts, pn);
}

size_t snn_b200_workspace_bytes(const snn_net_t *net0, const snn_run_opts_t *opts) {
    snn_net_t P;
    bool pn;
    if (strip_pn(net0, &P, &pn) != SNN_OK) return 0;
    const snn_net_t *net = &P;
    if (validate(net, opts) != SNN_OK) return 0;
    size_t g = layout_generic(net, opts, nullptr, nullptr);
    if (pn || has_sparse(net) || has_feat(net) || has_pool(net) || has_syn(net) || has_meanfield(net) || has_avg(net) || has_wn(net)) return g;
    size_t f = snn_fused_dc_supported(net, opts) ? snn_fused_dc_workspace_bytes(net, opts) : 0;
    size_t f2 = snn_fused_dc2_supported(net, opts) ? snn_fused_dc2_workspace_bytes(net, opts) : 0;
    if (f2 > f) f = f2;
    return g > f ? g : f;
}

int snn_b200_run_window(const snn_net_t *net0, const snn_run_opts_t *opts, void *workspace, size_t workspace_bytes,
                        void *stream_) {
    g_last_launches = 0;
    snn_net_t P;
    bool pn;
    int rc = strip_pn(net0, &P, &pn);
    if (rc != SNN_OK) return rc;
    const snn_net_t *net = &P;
    rc = validate(net, opts);
    if (rc != SNN_OK) return rc;
    cudaStream_t stream = (cudaStream_t)stream_;
    if (opts->T == 0 && !opts->normalize) return SNN_OK;
    const int tier = select_tier(net, opts, pn);
    if (tier == 0) return SNN_ERR_UNSUPPORTED;
    if (!workspace) return SNN_ERR_WORKSPACE;
    if (tier == 3) {
        if (workspace_bytes < snn_fused_dc2_workspace_bytes(net, opts)) return SNN_ERR_WORKSPACE;
        return snn_fused_dc2_launch(net, opts, workspace, workspace_bytes, stream, &g_last_launches);
    }
    if (tier == 2) {
        if (workspace_bytes < snn_fused_dc_workspace_bytes(net, opts)) return SNN_ERR_WORKSPACE;
        return snn_fused_dc_launch(net, opts, workspace, workspace_bytes, stream, &g_last_launches);
    }
    DevNet N;
    memset(&N, 0, sizeof(N));
    const size_t need = layout_generic(net, opts, (char *)workspace, &N);
    if (workspace_bytes < need) return SNN_ERR_WORKSPACE;
    N.n_layers = net->n_layers; N.n_conns = net->n_conns; N.learning = net->learning;
    N.T = opts->T; N.B = opts->B; N.normalize = opts->normalize;
    N.seed = opts->seed; N.step_offset = opts->step_offset; N.err = opts->err_flag;
    N.one_step = opts->one_step ? 1 : 0;
    for (int c = 0; c < net->n_conns; ++c) {
        N.conns[c] = net->conns[c];
        const snn_conn_t &C = net->conns[c];
        if (C.mask) N.any_mask = 1;
        if (C.kind == SNN_CONN_MCC && (C.f_prob || C.f_mask || C.f_int)) N.any_feat = 1;
    }
    N.any_pool = has_pool(net) ? 1 : 0;
    N.any_avg = has_avg(net) ? 1 : 0;
    N.any_wn = has_wn(net) ? 1 : 0;
    if (cudaMemsetAsync(N.bar, 0, sizeof(unsigned int) * SNN_BAR_ZERO_WORDS, stream) != cudaSuccess) return SNN_ERR_CUDA;
    const int e = snn_generic_launch(N, stream);
    if (e != 0) {
        fprintf(stderr, "libsnn_b200: generic window launch failed: %s\n", cudaGetErrorString((cudaError_t)e));
        return SNN_ERR_CUDA;
    }
    g_last_launches = 1;  // the persistent window kernel (the memset node is not ours)
    return SNN_OK;
}

}  // extern "C"
