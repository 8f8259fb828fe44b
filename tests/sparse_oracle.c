/*
 * sparse_oracle.c — TEST INFRASTRUCTURE: the CPU oracle (oracle/snn_oracle.c, included unchanged) extended by the
 * SparseConnection kind SNN_CONN_SPARSE (reference: topology.py:2009-2017).  It exports the oracle's own entry points
 * (snn_oracle_run_window, snn_oracle_conn_compute / conn_update / conn_normalize, snn_oracle_abi_version), so it is a
 * drop-in superset of libsnn_oracle.so: plans without a sparse connection go to the oracle's functions untouched.
 *
 * The sparse kind is restated over the CSR, never densified: p[b,j] = sum over the spiking i (ascending) of the stored
 * w[i,j], from +0, then + b[j] — `s.float() @ w + b` on a sparse w (topology.py:332-346); learning.NoOp's
 * `w *= weight_decay` (learning.py:93-94) scales the stored values, never clamped.  Same arithmetic contract as the
 * oracle (-ffp-contract=off, one rounding per reference op).
 *
 *   gcc -O2 -fPIC -std=c11 -ffp-contract=off -fno-fast-math -fopenmp -shared -o libsnn_sparse_oracle.so sparse_oracle.c -lm
 */
#define snn_oracle_run_window oracle_run_window_base
#define snn_oracle_conn_compute oracle_conn_compute_base
#define snn_oracle_conn_update oracle_conn_update_base
#define snn_oracle_conn_normalize oracle_conn_normalize_base
#include "../oracle/snn_oracle.c"
#undef snn_oracle_run_window
#undef snn_oracle_conn_compute
#undef snn_oracle_conn_update
#undef snn_oracle_conn_normalize

int snn_oracle_run_window(const snn_net_t *net, const snn_run_opts_t *o, int dense, int threads);
int snn_oracle_conn_compute(const snn_conn_t *C, int32_t n_src, int32_t n_tgt, int32_t B, const uint8_t *s, float *out);
int snn_oracle_conn_update(const snn_net_t *net, int32_t ci, int32_t B);
int snn_oracle_conn_normalize(const snn_conn_t *C, int32_t n_src, int32_t n_tgt);

/* 0 <= rowptr[i] <= rowptr[i+1] <= nnz, columns in [0, n_tgt), strictly ascending within a row (what coalesce() leaves);
 * a fixed pattern: rules NONE / NOOP only — the reference's other rules grow it (learning.py:403-417) or fail with finite
 * bounds (:101-102); normalize fails on a sparse w (aten::eq.Scalar), masks raise (topology.py:129-131). */
static int check_sparse(const snn_conn_t *C, int ns, int nt) {
    if (C->rule != SNN_RULE_NONE && C->rule != SNN_RULE_NOOP) return SNN_ERR_UNSUPPORTED;
    if (C->has_norm || C->mask) return SNN_ERR_UNSUPPORTED;
    if (C->nnz < 0 || !C->sp_rowptr || (C->nnz > 0 && (!C->sp_col || !C->w))) return SNN_ERR_BAD_ARG;
    for (int i = 0; i < ns; ++i) {
        const int a = C->sp_rowptr[i], e = C->sp_rowptr[i + 1];
        if (a < 0 || e < a || e > C->nnz) return SNN_ERR_BAD_ARG;
        for (int p = a; p < e; ++p)
            if (C->sp_col[p] < 0 || C->sp_col[p] >= nt || (p > a && C->sp_col[p] <= C->sp_col[p - 1])) return SNN_ERR_BAD_ARG;
    }
    return SNN_OK;
}

/* SparseConnection.compute, added into the target's accumulator like network.py:248 does.  `dense` = 1 visits the rows
 * of the silent sources too (adding 0 * w), the oracle's costed form. */
static void sparse_compute(const snn_conn_t *C, const snn_layer_t *S, int n_tgt, int B, float *cur, int dense) {
    const int ns = S->n;
#pragma omp parallel
    {
        float *p = (float *)malloc(sizeof(float) * (size_t)n_tgt);
#pragma omp for schedule(static)
        for (int b = 0; b < B; ++b) {
            const uint8_t *s = S->s + (size_t)b * ns;
            for (int j = 0; j < n_tgt; ++j) p[j] = 0.0f;
            for (int i = 0; i < ns; ++i) {
                if (!dense && !s[i]) continue;
                const float sv = s[i] ? 1.0f : 0.0f;
                for (int q = C->sp_rowptr[i]; q < C->sp_rowptr[i + 1]; ++q) p[C->sp_col[q]] = p[C->sp_col[q]] + sv * C->w[q];
            }
            float *cb = cur + (size_t)b * n_tgt;
            if (C->b)
                for (int j = 0; j < n_tgt; ++j) cb[j] = cb[j] + (p[j] + C->b[j]);   /* topology.py:345 */
            else
                for (int j = 0; j < n_tgt; ++j) cb[j] = cb[j] + p[j];
        }
        free(p);
    }
}

static void sparse_decay(const snn_conn_t *C) {
    if (C->rule != SNN_RULE_NOOP || C->weight_decay == 0.0f || C->weight_decay == 1.0f) return;
    for (int q = 0; q < C->nnz; ++q) C->w[q] = C->w[q] * C->weight_decay;
}

static void any_compute(const snn_net_t *net, const snn_conn_t *C, int B, float *cur, int dense) {
    const snn_layer_t *S = &net->layers[C->src];
    const int nt = net->layers[C->tgt].n;
    if (C->kind == SNN_CONN_CONV2D) conv_compute(C, S, B, cur, dense);
    else if (C->kind == SNN_CONN_SPARSE) sparse_compute(C, S, nt, B, cur, dense);
    else conn_compute(C, S, nt, B, cur, dense);
}

/* Network.run (network.py:252-465): oracle/snn_oracle.c's timestep loop, with the sparse kind in _get_inputs and in the
 * connection updates. */
int snn_oracle_run_window(const snn_net_t *net, const snn_run_opts_t *o, int dense, int threads) {
    if (!net || !o) return SNN_ERR_BAD_ARG;
    int any_sparse = 0;
    for (int c = 0; c < net->n_conns && c < SNN_MAX_CONNS; ++c) any_sparse |= net->conns[c].kind == SNN_CONN_SPARSE;
    if (!any_sparse) return oracle_run_window_base(net, o, dense, threads);
    /* the oracle's plan check, with each sparse connection presented as the dense connection it restates (its pointers
     * only: nothing is densified), then the pattern checks */
    snn_net_t probe = *net;
    float dummy = 0.0f;
    for (int c = 0; c < net->n_conns; ++c)
        if (probe.conns[c].kind == SNN_CONN_SPARSE) { probe.conns[c].kind = SNN_CONN_DENSE; probe.conns[c].w = &dummy; }
    int rc = check_plan(&probe, o);
    if (rc) return rc;
    for (int c = 0; c < net->n_conns; ++c) {
        const snn_conn_t *C = &net->conns[c];
        if (C->kind != SNN_CONN_SPARSE) continue;
        rc = check_sparse(C, net->layers[C->src].n, net->layers[C->tgt].n);
        if (rc) return rc;
    }
#ifdef _OPENMP
    if (threads > 0) omp_set_num_threads(threads);
#else
    (void)threads;
#endif
    const int B = o->B, T = o->T;
    layer_ws_t lws[SNN_MAX_LAYERS];
    conn_ws_t cws[SNN_MAX_CONNS];
    memset(lws, 0, sizeof(lws)); memset(cws, 0, sizeof(cws));
    for (int l = 0; l < net->n_layers; ++l) {
        const size_t BN = (size_t)B * net->layers[l].n;
        lws[l].cur = (float *)calloc(BN, sizeof(float));
        lws[l].cand = (uint8_t *)calloc(BN, 1);
    }
    for (int c = 0; c < net->n_conns; ++c) {
        const snn_conn_t *C = &net->conns[c];
        const int ns = net->layers[C->src].n, nt = net->layers[C->tgt].n;
        if (SNN_RULE_IS_STDP(C->rule) && C->kind != SNN_CONN_CONV2D) {
            cws[c].U = (float *)calloc((size_t)ns * nt, sizeof(float));
            cws[c].V = (float *)calloc((size_t)ns * nt, sizeof(float));
            cws[c].tx = (float *)calloc((size_t)B * nt, sizeof(float));
        }
        cws[c].row_t = (uint8_t *)calloc((size_t)ns, 1);
        cws[c].col_t = (uint8_t *)calloc((size_t)nt, 1);
    }
    int err = 0;
    for (int t = 0; t < T; ++t) {
        /* 1. _get_inputs (network.py:211-250): currents from the PREVIOUS step's spikes, in insertion order */
        for (int l = 0; l < net->n_layers; ++l) lws[l].has_in = 0;
        for (int c = 0; c < net->n_conns && !o->one_step; ++c) {
            const snn_conn_t *C = &net->conns[c];
            const snn_layer_t *G = &net->layers[C->tgt];
            if (!lws[C->tgt].has_in) { memset(lws[C->tgt].cur, 0, sizeof(float) * (size_t)B * G->n); lws[C->tgt].has_in = 1; }
            any_compute(net, C, B, lws[C->tgt].cur, dense);
        }
        /* 2. layers in insertion order (network.py:386-429); one-step mode recomputes a layer's input just before it */
        for (int l = 0; l < net->n_layers; ++l) {
            if (o->one_step)
                for (int c = 0; c < net->n_conns; ++c) {
                    const snn_conn_t *C = &net->conns[c];
                    if (C->tgt != l) continue;
                    if (!lws[l].has_in) { memset(lws[l].cur, 0, sizeof(float) * (size_t)B * net->layers[l].n); lws[l].has_in = 1; }
                    any_compute(net, C, B, lws[l].cur, dense);
                }
            layer_forward(net, l, o, t, &lws[l], &err);
        }
        /* 3. connection updates in insertion order (network.py:431-454) */
        if (net->learning)
            for (int c = 0; c < net->n_conns; ++c) {
                const snn_conn_t *C = &net->conns[c];
                if (C->kind == SNN_CONN_SPARSE) sparse_decay(C);
                else if (C->rule == SNN_RULE_MSTDP && C->kind == SNN_CONN_CONV2D) mstdp_conv_update(net, C, o, dense);
                else if (C->rule == SNN_RULE_MSTDP) mstdp_dense_update(net, C, o, dense);
                else if (C->rule == SNN_RULE_MSTDPET) mstdpet_dense_update(net, C);
                else if (C->kind == SNN_CONN_CONV2D && SNN_RULE_IS_STDP(C->rule)) stdp_conv_update(net, C, o, dense);
                else if (C->kind == SNN_CONN_CONV2D) {
                    if (C->rule == SNN_RULE_NOOP && C->weight_decay != 0.0f)
                        for (size_t k = 0; k < (size_t)C->cout * C->cin * C->kh * C->kw; ++k) C->w[k] = C->w[k] * C->weight_decay;
                } else conn_update(net, C, o, &cws[c], dense);
            }
        /* connection masks (topology.py:127-131): dense connections only */
        for (int c = 0; c < net->n_conns; ++c) {
            const snn_conn_t *C = &net->conns[c];
            if (!C->mask || C->kind != SNN_CONN_DENSE) continue;
            const size_t NW = (size_t)net->layers[C->src].n * net->layers[C->tgt].n;
            for (size_t k = 0; k < NW; ++k) if (C->mask[k]) C->w[k] = 0.0f;
        }
        /* 4. monitors (network.py:460-461, monitors.py:94-111) */
        for (int l = 0; l < net->n_layers; ++l) {
            const snn_layer_t *L = &net->layers[l];
            const size_t BN = (size_t)B * L->n;
            if (L->rec_s) memcpy(L->rec_s + (size_t)t * BN, L->s, BN);
            if (L->rec_v && L->v) memcpy(L->rec_v + (size_t)t * BN, L->v, BN * sizeof(float));
            if (L->rec_count) for (size_t k = 0; k < BN; ++k) L->rec_count[k] += L->s[k] ? 1 : 0;
        }
    }
    /* network.py:464-465 (a sparse connection never has has_norm: checked above) */
    if (o->normalize)
        for (int c = 0; c < net->n_conns; ++c) {
            const snn_conn_t *C = &net->conns[c];
            if (C->has_norm && C->kind == SNN_CONN_CONV2D) normalize_conv(C);
            else if (C->has_norm) normalize_cols(C->w, net->layers[C->src].n, net->layers[C->tgt].n, C->norm_abs, C->norm);
        }
    for (int l = 0; l < net->n_layers; ++l) { free(lws[l].cur); free(lws[l].cand); }
    for (int c = 0; c < net->n_conns; ++c) { free(cws[c].U); free(cws[c].V); free(cws[c].tx); free(cws[c].row_t); free(cws[c].col_t); }
    if (o->err_flag) *o->err_flag |= err;
    return SNN_OK;
}

int snn_oracle_conn_compute(const snn_conn_t *C, int32_t n_src, int32_t n_tgt, int32_t B, const uint8_t *s, float *out) {
    if (!C || C->kind != SNN_CONN_SPARSE) return oracle_conn_compute_base(C, n_src, n_tgt, B, s, out);
    if (!s || !out) return SNN_ERR_BAD_ARG;
    snn_conn_t probe = *C;
    probe.rule = SNN_RULE_NONE;   /* compute does not involve the rule */
    int rc = check_sparse(&probe, n_src, n_tgt);
    if (rc) return rc;
    snn_layer_t S; memset(&S, 0, sizeof(S)); S.n = n_src; S.s = (uint8_t *)s;
    memset(out, 0, sizeof(float) * (size_t)B * n_tgt);
    sparse_compute(C, &S, n_tgt, B, out, 0);
    return SNN_OK;
}

int snn_oracle_conn_update(const snn_net_t *net, int32_t ci, int32_t B) {
    if (!net || ci < 0 || ci >= net->n_conns || net->conns[ci].kind != SNN_CONN_SPARSE) return oracle_conn_update_base(net, ci, B);
    const snn_conn_t *C = &net->conns[ci];
    if (C->rule != SNN_RULE_NONE && C->rule != SNN_RULE_NOOP) return SNN_ERR_UNSUPPORTED;
    sparse_decay(C);
    return SNN_OK;
}

int snn_oracle_conn_normalize(const snn_conn_t *C, int32_t n_src, int32_t n_tgt) {
    if (C && C->kind == SNN_CONN_SPARSE) return SNN_ERR_UNSUPPORTED;   /* aten::eq.Scalar has no SparseCPU kernel */
    return oracle_conn_normalize_base(C, n_src, n_tgt);
}
