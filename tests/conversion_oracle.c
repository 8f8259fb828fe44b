/*
 * conversion_oracle.c — TEST INFRASTRUCTURE: the max-pooling oracle (tests/maxpool_oracle.c, which includes the CPU
 * oracle oracle/snn_oracle.c; both included unchanged) extended by the two layer kinds ann_to_snn emits besides the
 * built-in ones: SubtractiveResetIFNodes (SNN_NODE_SUBIF) and PassThroughNodes (SNN_NODE_PASSTHROUGH).  It exports the
 * oracle's own entry points, so it is a drop-in superset of libsnn_maxpool_oracle.so: plans without such a layer go to
 * the max-pooling oracle's window untouched.
 *
 * SubtractiveResetIFNodes.forward (conversion/nodes.py:73-99), one rounding per op:
 *   v  = v + (rc == 0).float() * x
 *   rc = (rc > 0).float() * (rc - dt)
 *   s  = v >= thresh;  where s: rc = refrac, v = v - thresh
 *   v  = lbound where v < lbound (if lbound is given);  then Nodes.forward: traces, summed += x
 * PassThroughNodes.forward (:137-144): s = x — no trace, no summed input.  Its s is float32 in the plan (include/
 * snn_b200.h); this oracle keeps a 0 / 1 byte copy of it for the step, so that the oracle's connection, learning and
 * recording code reads it as it reads every other layer's spikes, and writes the float back at the end.  A value
 * outside {0, 1} raises SNN_ERR_NONBINARY.
 *
 *   gcc -O2 -fPIC -std=c11 -ffp-contract=off -fno-fast-math -fopenmp -shared -o libsnn_conversion_oracle.so conversion_oracle.c -lm
 */
#include "../include/snn_b200.h"

/* The max-pooling oracle's window keeps its code but not its symbol; the window below takes the exported one. */
int snn_oracle_run_window(const snn_net_t *net, const snn_run_opts_t *o, int dense, int threads) __asm__("maxpool_oracle_run_window");
#include "maxpool_oracle.c"

int conversion_run_window(const snn_net_t *net, const snn_run_opts_t *o, int dense, int threads) __asm__("snn_oracle_run_window");

static int is_conversion_kind(int kind) { return kind == SNN_NODE_SUBIF || kind == SNN_NODE_PASSTHROUGH; }

/* include/snn_b200.h's conditions on the two kinds, then the oracle's own checks (with the pooling connections checked
 * by pool_check) on the plan in which a SubtractiveResetIFNodes layer stands for an IFNodes one (the same state) and a
 * PassThroughNodes layer for a stateless McCullochPitts one. */
static int conversion_check_plan(const snn_net_t *net, const snn_run_opts_t *o) {
    static snn_net_t rest;   /* large for the stack; the oracle runs one window at a time */
    static float dummy;
    if (net->n_layers < 1 || net->n_layers > SNN_MAX_LAYERS || net->n_conns < 0 || net->n_conns > SNN_MAX_CONNS) return SNN_ERR_BAD_ARG;
    memcpy(&rest, net, sizeof(rest));
    rest.n_conns = 0;
    for (int l = 0; l < net->n_layers; ++l) {
        snn_layer_t *L = &rest.layers[l];
        if (L->kind == SNN_NODE_SUBIF) L->kind = SNN_NODE_IF;
        if (L->kind == SNN_NODE_PASSTHROUGH) {
            L->kind = SNN_NODE_MCP;
            L->v = &dummy;
            L->traces = L->sum_input = 0;
        }
    }
    for (int c = 0; c < net->n_conns; ++c) {
        const snn_conn_t *C = &net->conns[c];
        if (C->src < 0 || C->src >= net->n_layers || C->tgt < 0 || C->tgt >= net->n_layers) return SNN_ERR_BAD_ARG;
        const int ps = net->layers[C->src].kind == SNN_NODE_PASSTHROUGH, pt = net->layers[C->tgt].kind == SNN_NODE_PASSTHROUGH;
        if (pt && C->kind != SNN_CONN_MAXPOOL2D) return SNN_ERR_UNSUPPORTED;
        if ((ps || pt) && C->rule != SNN_RULE_NONE && C->rule != SNN_RULE_NOOP) return SNN_ERR_UNSUPPORTED;
        if (C->kind != SNN_CONN_MAXPOOL2D) { rest.conns[rest.n_conns++] = *C; continue; }
        if (net->layers[C->tgt].kind == SNN_NODE_INPUT) return SNN_ERR_UNSUPPORTED;
        const int rc = pool_check(C, net->layers[C->src].n, net->layers[C->tgt].n);
        if (rc) return rc;
    }
    return check_plan(&rest, o);
}

/* network.py:386-413: the layer's input of step t — the connections' sum (zero without one) plus the external input,
 * which one-step mode drops for a layer with an incoming connection. */
static void layer_input(const snn_layer_t *L, const snn_run_opts_t *o, int t, layer_ws_t *ws) {
    const size_t BN = (size_t)o->B * L->n;
    if (!ws->has_in) memset(ws->cur, 0, sizeof(float) * BN);
    if (o->one_step && ws->has_in) return;
    if (L->ext_dtype == SNN_EXT_U8) {
        const uint8_t *e = (const uint8_t *)L->ext + (size_t)t * BN;
        for (size_t k = 0; k < BN; ++k) ws->cur[k] = ws->cur[k] + (float)e[k];
    } else if (L->ext_dtype == SNN_EXT_F32) {
        const float *e = (const float *)L->ext + (size_t)t * BN;
        for (size_t k = 0; k < BN; ++k) ws->cur[k] = ws->cur[k] + e[k];
    }
}

/* network.py:415-429: clamp / unclamp after forward. */
static void clamp_spikes(const snn_layer_t *L, int B, int t) {
    const int n = L->n;
    if (L->clamp) {
        const uint8_t *m = L->clamp + (L->clamp_per_step ? (size_t)t * n : 0);
        for (int b = 0; b < B; ++b)
            for (int j = 0; j < n; ++j) if (m[j]) L->s[(size_t)b * n + j] = 1;
    }
    if (L->unclamp) {
        const uint8_t *m = L->unclamp + (L->unclamp_per_step ? (size_t)t * n : 0);
        for (int b = 0; b < B; ++b)
            for (int j = 0; j < n; ++j) if (m[j]) L->s[(size_t)b * n + j] = 0;
    }
}

/* One step of a layer of either kind; `L` is the byte view (a PassThroughNodes layer's s is the byte copy). */
static void conversion_forward(const snn_layer_t *L, const snn_run_opts_t *o, int t, layer_ws_t *ws, int *err) {
    const int B = o->B, n = L->n;
    const size_t BN = (size_t)B * n;
    layer_input(L, o, t, ws);
    const float *cur = ws->cur;
    if (L->kind == SNN_NODE_PASSTHROUGH) {
        for (size_t k = 0; k < BN; ++k) {
            L->s[k] = cur[k] != 0.0f;
            if (cur[k] != 0.0f && cur[k] != 1.0f) *err |= SNN_ERR_NONBINARY;
        }
    } else {
        if (L->inject_v) {   /* network.py:398-404 */
            const float *iv = L->inject_v + (L->inject_per_step ? (size_t)t * n : 0);
            for (int b = 0; b < B; ++b)
                for (int j = 0; j < n; ++j) L->v[(size_t)b * n + j] += iv[j];
        }
        for (size_t k = 0; k < BN; ++k) {
            float v = L->v[k], rc = L->refrac_count[k];
            const float gate = rc == 0.0f ? 1.0f : 0.0f;
            v = v + gate * cur[k];                                    /* :82 */
            const float keep = rc > 0.0f ? 1.0f : 0.0f;
            rc = keep * (rc - L->dt);                                 /* :85-87 */
            const int s = v >= L->thresh;                             /* :90 */
            if (s) { rc = L->refrac; v = v - L->thresh; }             /* :93-94 */
            if (L->has_lbound && v < L->lbound) v = L->lbound;        /* :97-98 */
            L->v[k] = v; L->refrac_count[k] = rc; L->s[k] = (uint8_t)s;
            trace_and_sum(L, k, s, cur[k]);                           /* :99 */
        }
    }
    clamp_spikes(L, B, t);
}

/* Network.run (network.py:252-465): tests/maxpool_oracle.c's timestep loop with the two kinds in the layer pass. */
int conversion_run_window(const snn_net_t *net, const snn_run_opts_t *o, int dense, int threads) {
    if (!net || !o) return SNN_ERR_BAD_ARG;
    int any = 0;
    for (int l = 0; l < net->n_layers && l < SNN_MAX_LAYERS; ++l) any |= is_conversion_kind(net->layers[l].kind);
    if (!any) return snn_oracle_run_window(net, o, dense, threads);
    int rc = conversion_check_plan(net, o);
    if (rc) return rc;
#ifdef _OPENMP
    if (threads > 0) omp_set_num_threads(threads);
#endif
    const int B = o->B, T = o->T;
    static snn_net_t v8;   /* the plan with every PassThroughNodes layer's s replaced by its byte copy */
    memcpy(&v8, net, sizeof(v8));
    int err = 0;
    for (int l = 0; l < net->n_layers; ++l) {
        const snn_layer_t *L = &net->layers[l];
        if (L->kind != SNN_NODE_PASSTHROUGH) continue;
        const size_t BN = (size_t)B * L->n;
        const float *f = (const float *)L->s;
        uint8_t *s8 = (uint8_t *)malloc(BN);
        for (size_t k = 0; k < BN; ++k) {
            s8[k] = f[k] != 0.0f;
            if (f[k] != 0.0f && f[k] != 1.0f) err |= SNN_ERR_NONBINARY;
        }
        v8.layers[l].s = s8;
    }
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
    for (int t = 0; t < T; ++t) {
        /* 1. _get_inputs (network.py:211-250): currents from the PREVIOUS step's spikes, in insertion order */
        for (int l = 0; l < net->n_layers; ++l) lws[l].has_in = 0;
        for (int c = 0; c < net->n_conns && !o->one_step; ++c) {
            const snn_conn_t *C = &net->conns[c];
            if (!lws[C->tgt].has_in) { memset(lws[C->tgt].cur, 0, sizeof(float) * (size_t)B * net->layers[C->tgt].n); lws[C->tgt].has_in = 1; }
            any_compute(&v8, c, o, lws[C->tgt].cur, dense);
        }
        /* 2. layers in insertion order (network.py:386-429); one-step mode recomputes a layer's input just before it */
        for (int l = 0; l < net->n_layers; ++l) {
            if (o->one_step)
                for (int c = 0; c < net->n_conns; ++c) {
                    if (net->conns[c].tgt != l) continue;
                    if (!lws[l].has_in) { memset(lws[l].cur, 0, sizeof(float) * (size_t)B * net->layers[l].n); lws[l].has_in = 1; }
                    any_compute(&v8, c, o, lws[l].cur, dense);
                }
            if (is_conversion_kind(v8.layers[l].kind)) conversion_forward(&v8.layers[l], o, t, &lws[l], &err);
            else layer_forward(&v8, l, o, t, &lws[l], &err);
        }
        /* 3. connection updates in insertion order (network.py:431-454) */
        if (net->learning)
            for (int c = 0; c < net->n_conns; ++c) {
                const snn_conn_t *C = &net->conns[c];
                if (C->kind == SNN_CONN_MAXPOOL2D) continue;
                if (C->rule == SNN_RULE_MSTDP && C->kind == SNN_CONN_CONV2D) mstdp_conv_update(&v8, C, o, dense);
                else if (C->rule == SNN_RULE_MSTDP) mstdp_dense_update(&v8, C, o, dense);
                else if (C->rule == SNN_RULE_MSTDPET) mstdpet_dense_update(&v8, C);
                else if (C->kind == SNN_CONN_CONV2D && SNN_RULE_IS_STDP(C->rule)) stdp_conv_update(&v8, C, o, dense);
                else if (C->kind == SNN_CONN_CONV2D) {
                    if (C->rule == SNN_RULE_NOOP && C->weight_decay != 0.0f)
                        for (size_t k = 0; k < (size_t)C->cout * C->cin * C->kh * C->kw; ++k) C->w[k] = C->w[k] * C->weight_decay;
                } else conn_update(&v8, C, o, &cws[c], dense);
            }
        for (int c = 0; c < net->n_conns; ++c) {   /* connection masks (topology.py:127-131): dense connections only */
            const snn_conn_t *C = &net->conns[c];
            if (!C->mask || C->kind != SNN_CONN_DENSE) continue;
            const size_t NW = (size_t)net->layers[C->src].n * net->layers[C->tgt].n;
            for (size_t k = 0; k < NW; ++k) if (C->mask[k]) C->w[k] = 0.0f;
        }
        /* 4. monitors (network.py:460-461, monitors.py:94-111) */
        for (int l = 0; l < net->n_layers; ++l) {
            const snn_layer_t *L = &v8.layers[l];
            const size_t BN = (size_t)B * L->n;
            if (L->rec_s) memcpy(L->rec_s + (size_t)t * BN, L->s, BN);
            if (L->rec_v && L->v) memcpy(L->rec_v + (size_t)t * BN, L->v, BN * sizeof(float));
            if (L->rec_count) for (size_t k = 0; k < BN; ++k) L->rec_count[k] += L->s[k] ? 1 : 0;
        }
    }
    if (o->normalize)   /* network.py:464-465 */
        for (int c = 0; c < net->n_conns; ++c) {
            const snn_conn_t *C = &net->conns[c];
            if (C->kind == SNN_CONN_MAXPOOL2D || !C->has_norm) continue;
            if (C->kind == SNN_CONN_CONV2D) normalize_conv(C);
            else normalize_cols(C->w, net->layers[C->src].n, net->layers[C->tgt].n, C->norm_abs, C->norm);
        }
    for (int l = 0; l < net->n_layers; ++l) {
        free(lws[l].cur); free(lws[l].cand);
        if (net->layers[l].kind != SNN_NODE_PASSTHROUGH) continue;
        float *f = (float *)net->layers[l].s;
        const uint8_t *s8 = v8.layers[l].s;
        if (T > 0)
            for (size_t k = 0; k < (size_t)B * net->layers[l].n; ++k) f[k] = s8[k] ? 1.0f : 0.0f;
        free(v8.layers[l].s);
    }
    for (int c = 0; c < net->n_conns; ++c) { free(cws[c].U); free(cws[c].V); free(cws[c].tx); free(cws[c].row_t); free(cws[c].col_t); }
    if (o->err_flag) *o->err_flag |= err;
    return SNN_OK;
}
