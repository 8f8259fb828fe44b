/*
 * weight_norm_oracle.c — TEST INFRASTRUCTURE: the feature oracle (tests/feature_oracle.c, which includes the CPU oracle
 * oracle/snn_oracle.c; both included unchanged) extended by per-target norm tensors and per-step Weight normalisation
 * (SNN_CONN_WNORM, include/snn_b200.h).  It exports the oracle's own entry points, so it is a drop-in superset of
 * libsnn_feature_oracle.so: plans without the flag go to the feature oracle's window and normalize untouched.
 *
 * Weight(norm_frequency='time step') normalises inside Weight.compute, after the product (topology_features.py:633-645):
 * here right after the step's inputs are gathered, before the rules run; the rule's clamp then reaches every element
 * (MCC_learning.py:101-110), which the oracle's event-driven update does not visit, so a clamp pass over the whole
 * matrix follows it.  The factor of a column is the one the header states for each form of the norm, the column sum is
 * taken in the SNN_NORM_CHUNKS order.  MCC_learning.MSTDP / MSTDPET run as the oracle's dense rules, as in
 * tests/mcc_reward_oracle.c.
 *
 *   gcc -O2 -fPIC -std=c11 -ffp-contract=off -fno-fast-math -fopenmp -shared -o libsnn_weight_norm_oracle.so weight_norm_oracle.c -lm
 */
#include "../include/snn_b200.h"

/* The feature oracle's window and normalize keep their code but not their symbols: these declarations give them other
 * assembler names, and the functions below take the exported ones. */
int snn_oracle_run_window(const snn_net_t *net, const snn_run_opts_t *o, int dense, int threads) __asm__("feature_oracle_run_window");
int snn_oracle_conn_normalize(const snn_conn_t *C, int32_t n_src, int32_t n_tgt) __asm__("feature_oracle_conn_normalize");
int snn_oracle_conn_compute(const snn_conn_t *C, int32_t n_src, int32_t n_tgt, int32_t B, const uint8_t *s, float *out)
    __asm__("feature_oracle_conn_compute");
#include "feature_oracle.c"

int weight_norm_run_window(const snn_net_t *net, const snn_run_opts_t *o, int dense, int threads) __asm__("snn_oracle_run_window");
int weight_norm_conn_normalize(const snn_conn_t *C, int32_t n_src, int32_t n_tgt) __asm__("snn_oracle_conn_normalize");
int weight_norm_conn_compute(const snn_conn_t *C, int32_t n_src, int32_t n_tgt, int32_t B, const uint8_t *s, float *out)
    __asm__("snn_oracle_conn_compute");

/* compute(): the product does not read the norm (the caller normalises after it), so the flag is dropped */
int weight_norm_conn_compute(const snn_conn_t *C, int32_t n_src, int32_t n_tgt, int32_t B, const uint8_t *s, float *out) {
    if (!C || !(C->kind & SNN_CONN_WNORM)) return feature_oracle_conn_compute(C, n_src, n_tgt, B, s, out);
    snn_conn_t K = *C;
    K.kind &= ~SNN_CONN_WNORM;
    return feature_oracle_conn_compute(&K, n_src, n_tgt, B, s, out);
}

/* The flag's fields (the library's checks): a dense or MCC connection with a norm, a per-step flag on an MCC Weight only,
 * no averaged rule. */
static int wn_fields_ok(const snn_conn_t *C) {
    const int kind = C->kind & ~SNN_CONN_WNORM;
    if (kind != SNN_CONN_DENSE && kind != SNN_CONN_MCC) return SNN_ERR_UNSUPPORTED;
    if (!C->has_norm || (C->norm_step != 0 && C->norm_step != 1)) return SNN_ERR_BAD_ARG;
    if ((C->norm_step && kind != SNN_CONN_MCC) || (C->rule & SNN_RULE_AVG)) return SNN_ERR_UNSUPPORTED;
    return SNN_OK;
}

/* w[:, j] *= f[j] with the factor of the norm's form (snn_b200.h SNN_CONN_WNORM) */
static void wn_normalize(const snn_conn_t *C, int ns, int nt) {
    const int chunk = (ns + SNN_NORM_CHUNKS - 1) / SNN_NORM_CHUNKS;
#pragma omp parallel for schedule(static)
    for (int j = 0; j < nt; ++j) {
        float tot = 0.0f;
        for (int c = 0; c < SNN_NORM_CHUNKS; ++c) {
            float part = 0.0f;
            const int i1 = (c + 1) * chunk < ns ? (c + 1) * chunk : ns;
            for (int i = c * chunk; i < i1; ++i) {
                const float x = C->w[(size_t)i * nt + j];
                part = part + (C->norm_abs ? fabsf(x) : x);
            }
            tot = tot + part;
        }
        if (tot == 0.0f) tot = 1.0f;
        float f;
        if (C->norm_t) f = C->norm_t[j] / tot;                   /* Tensor / Tensor */
        else if (C->norm_step) { const float r = 1.0f / tot; f = r * C->norm; }   /* float / Tensor: reciprocal, then * norm */
        else f = C->norm / tot;
        for (int i = 0; i < ns; ++i) C->w[(size_t)i * nt + j] = C->w[(size_t)i * nt + j] * f;
    }
}

int weight_norm_run_window(const snn_net_t *net, const snn_run_opts_t *o, int dense, int threads) {
    if (!net || !o) return SNN_ERR_BAD_ARG;
    if (net->n_conns < 0 || net->n_conns > SNN_MAX_CONNS) return SNN_ERR_BAD_ARG;
    int any = 0;
    for (int c = 0; c < net->n_conns; ++c) any |= (net->conns[c].kind & SNN_CONN_WNORM) != 0;
    if (!any) return feature_oracle_run_window(net, o, dense, threads);
    static snn_net_t plain;   /* large for the stack; the oracle runs one window at a time */
    memcpy(&plain, net, sizeof(plain));
    int step_conn[SNN_MAX_CONNS] = {0};
    for (int c = 0; c < net->n_conns; ++c) {
        snn_conn_t *C = &plain.conns[c];
        if (!(C->kind & SNN_CONN_WNORM)) continue;
        const int rc = wn_fields_ok(C);
        if (rc) return rc;
        C->kind &= ~SNN_CONN_WNORM;
        step_conn[c] = C->norm_step;
        if (has_features(C) && C->kind != SNN_CONN_MCC) return SNN_ERR_BAD_ARG;
    }
    net = &plain;
    /* MCC_learning.MSTDP / MSTDPET are op for op the dense rules on the Weight's value (tests/mcc_reward_oracle.c): the
     * plan is checked as the oracle checks them on a dense Connection, and the window applies the dense updates */
    static snn_net_t as_dense;
    memcpy(&as_dense, &plain, sizeof(as_dense));
    for (int c = 0; c < net->n_conns; ++c)
        if (as_dense.conns[c].kind == SNN_CONN_MCC && SNN_RULE_IS_MSTDP(as_dense.conns[c].rule)) as_dense.conns[c].kind = SNN_CONN_DENSE;
    int rc = check_plan(&as_dense, o);
    if (rc) return rc;
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
            any_compute(net, c, o, t, lws[C->tgt].cur, dense);
            if (step_conn[c]) wn_normalize(C, net->layers[C->src].n, G->n);   /* Weight.compute's normalize */
        }
        /* 2. layers in insertion order (network.py:386-429); one-step mode recomputes a layer's input just before it */
        for (int l = 0; l < net->n_layers; ++l) {
            if (o->one_step)
                for (int c = 0; c < net->n_conns; ++c) {
                    const snn_conn_t *C = &net->conns[c];
                    if (C->tgt != l) continue;
                    if (!lws[l].has_in) { memset(lws[l].cur, 0, sizeof(float) * (size_t)B * net->layers[l].n); lws[l].has_in = 1; }
                    any_compute(net, c, o, t, lws[l].cur, dense);
                    if (step_conn[c]) wn_normalize(C, net->layers[C->src].n, net->layers[l].n);
                }
            layer_forward(net, l, o, t, &lws[l], &err);
        }
        /* 3. connection updates in insertion order (network.py:431-454); the rules read the Weight only */
        if (net->learning)
            for (int c = 0; c < net->n_conns; ++c) {
                const snn_conn_t *C = &net->conns[c];
                if (C->rule == SNN_RULE_MSTDP && C->kind == SNN_CONN_CONV2D) mstdp_conv_update(net, C, o, dense);
                else if (C->rule == SNN_RULE_MSTDP) mstdp_dense_update(net, C, o, dense);
                else if (C->rule == SNN_RULE_MSTDPET) mstdpet_dense_update(net, C);
                else if (C->kind == SNN_CONN_CONV2D && SNN_RULE_IS_STDP(C->rule)) stdp_conv_update(net, C, o, dense);
                else if (C->kind == SNN_CONN_CONV2D) {
                    if (C->rule == SNN_RULE_NOOP && C->weight_decay != 0.0f)
                        for (size_t k = 0; k < (size_t)C->cout * C->cin * C->kh * C->kw; ++k) C->w[k] = C->w[k] * C->weight_decay;
                } else conn_update(net, C, o, &cws[c], dense);
                /* the rule's clamp reaches every element of a Weight normalised this step (MCC_learning.py:101-110) */
                if (step_conn[c] && C->has_clamp && C->rule != SNN_RULE_NONE) {
                    const size_t NW = (size_t)net->layers[C->src].n * net->layers[C->tgt].n;
                    for (size_t k = 0; k < NW; ++k) C->w[k] = clampf(C->w[k], C->wmin, C->wmax);
                }
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
    /* network.py:464-465: a 'time step' Weight's normalize does nothing here (topology_features.py:663-671) */
    if (o->normalize)
        for (int c = 0; c < net->n_conns; ++c) {
            const snn_conn_t *C = &net->conns[c];
            if (!C->has_norm || step_conn[c]) continue;
            if (C->kind == SNN_CONN_CONV2D) normalize_conv(C);
            else wn_normalize(C, net->layers[C->src].n, net->layers[C->tgt].n);
        }
    for (int l = 0; l < net->n_layers; ++l) { free(lws[l].cur); free(lws[l].cand); }
    for (int c = 0; c < net->n_conns; ++c) { free(cws[c].U); free(cws[c].V); free(cws[c].tx); free(cws[c].row_t); free(cws[c].col_t); }
    if (o->err_flag) *o->err_flag |= err;
    return SNN_OK;
}

/* normalize() of one connection: a norm tensor, or the per-step formula when norm_step is set */
int weight_norm_conn_normalize(const snn_conn_t *C, int32_t n_src, int32_t n_tgt) {
    if (!C || !(C->kind & SNN_CONN_WNORM)) return feature_oracle_conn_normalize(C, n_src, n_tgt);
    const int kind = C->kind & ~SNN_CONN_WNORM;
    if (kind != SNN_CONN_DENSE && kind != SNN_CONN_MCC) return SNN_ERR_UNSUPPORTED;
    if (!C->w || (C->norm_step != 0 && C->norm_step != 1)) return SNN_ERR_BAD_ARG;
    if (C->has_norm) wn_normalize(C, n_src, n_tgt);
    return SNN_OK;
}
