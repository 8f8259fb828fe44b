/*
 * neuron_param_oracle.c — TEST INFRASTRUCTURE: the synapse-tensor oracle (tests/synapse_oracle.c, which includes the CPU
 * oracle oracle/snn_oracle.c; both included unchanged) extended by per-neuron parameters of LIFNodes, AdaptiveLIFNodes
 * and DiehlAndCookNodes layers (include/snn_b200.h SNN_NODE_PN: a parameter given as a tensor, which the reference
 * broadcasts elementwise against [B, *shape]).  It exports the oracle's own entry points, so it is a drop-in superset of
 * libsnn_synapse_oracle.so: plans without such a layer go to that oracle's window untouched.
 *
 * Each layer step below is the oracle's own (layer_forward), op for op, with neuron j's row of the block where the
 * oracle reads a scalar:
 *   LIF    v = fl(decay[j] * fl(v - rest[j])) + rest[j];  s = v >= thresh[j]                   (nodes.py:500-529)
 *   DC     theta[j] *= theta_decay[j];  s = v >= fl(thresh[j] + theta[j]);
 *          theta[j] += fl(theta_plus[j] * count)                                              (nodes.py:1069-1111)
 *   traces x = x * trace_decay[j];  x = x + fl(trace_scale[j] * s)  (additive only)           (nodes.py:96-103)
 *
 *   gcc -O2 -fPIC -std=c11 -ffp-contract=off -fno-fast-math -fopenmp -shared -o libsnn_neuron_param_oracle.so neuron_param_oracle.c -lm
 */
#include "../include/snn_b200.h"
#include <math.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

/* The synapse-tensor oracle's window and single-operator update, and the oracle's, keep their code under other names
 * (their assembler labels dropped, the oracle's entry points renamed); the functions below take the exported names. */
#define __asm__(label)
#define snn_oracle_run_window base_oracle_run_window
#define snn_oracle_conn_update base_oracle_conn_update
#include "synapse_oracle.c"
#undef snn_oracle_run_window
#undef snn_oracle_conn_update
#undef __asm__

/* include/snn_b200.h's conditions on the block */
static int pn_check(const snn_layer_t *L) {
    const int kind = L->kind & ~SNN_NODE_PN;
    if (kind != SNN_NODE_LIF && kind != SNN_NODE_DC) return SNN_ERR_BAD_ARG;
    uint32_t allowed = 1u << SNN_PN_THRESH | 1u << SNN_PN_REST | 1u << SNN_PN_DECAY;
    if (kind == SNN_NODE_DC) allowed |= 1u << SNN_PN_THETA_PLUS | 1u << SNN_PN_THETA_DECAY;
    if (L->traces) allowed |= 1u << SNN_PN_TRACE_DECAY;
    if (L->traces && L->traces_additive) allowed |= 1u << SNN_PN_TRACE_SCALE;
    if ((L->pn_mask & ~allowed) || (L->pn_mask && !L->pn)) return SNN_ERR_BAD_ARG;
    return SNN_OK;
}

/* neuron j's value of parameter `row` */
static inline float par(const snn_layer_t *L, int row, float scalar, int j) {
    return (L->pn_mask >> row) & 1u ? L->pn[(size_t)row * L->n + j] : scalar;
}

static inline void pn_trace_and_sum(const snn_layer_t *L, size_t k, int j, int s, float xin) {
    if (L->traces) {
        float x = L->x[k] * par(L, SNN_PN_TRACE_DECAY, L->trace_decay, j);                       /* nodes.py:98  */
        if (L->traces_additive) x = x + par(L, SNN_PN_TRACE_SCALE, L->trace_scale, j) * (s ? 1.0f : 0.0f); /* :101 */
        else if (s) x = L->trace_scale;                                                         /* :103 */
        L->x[k] = x;
    }
    if (L->sum_input) L->summed[k] = L->summed[k] + xin;                                        /* :107 */
}

/* layer_forward (oracle/snn_oracle.c) of an SNN_NODE_LIF / SNN_NODE_DC layer with a per-neuron block */
static void pn_layer_forward(const snn_net_t *net, int l, const snn_run_opts_t *o, int t, layer_ws_t *ws) {
    const snn_layer_t *L = &net->layers[l];
    const int B = o->B, n = L->n;
    const size_t BN = (size_t)B * n;
    float *cur = ws->cur;
    if (!ws->has_in) memset(cur, 0, sizeof(float) * BN);
    const int drop_ext = o->one_step && ws->has_in;
    if (drop_ext) {
    } else if (L->ext_dtype == SNN_EXT_U8) {
        const uint8_t *e = (const uint8_t *)L->ext + (size_t)t * BN;
        for (size_t k = 0; k < BN; ++k) cur[k] = cur[k] + (float)e[k];
    } else if (L->ext_dtype == SNN_EXT_F32) {
        const float *e = (const float *)L->ext + (size_t)t * BN;
        for (size_t k = 0; k < BN; ++k) cur[k] = cur[k] + e[k];
    }
    if (L->inject_v) {
        const float *iv = L->inject_v + (L->inject_per_step ? (size_t)t * n : 0);
        for (int b = 0; b < B; ++b)
            for (int j = 0; j < n; ++j) L->v[(size_t)b * n + j] += iv[j];
    }
    if (L->kind == SNN_NODE_LIF) {
        for (size_t k = 0; k < BN; ++k) {
            const int j = (int)(k % (size_t)n);
            const float rest = par(L, SNN_PN_REST, L->rest, j);
            float v = par(L, SNN_PN_DECAY, L->decay, j) * (L->v[k] - rest) + rest;   /* :508 */
            float xin = cur[k];
            if (L->refrac_count[k] > 0.0f) xin = 0.0f;
            float rc = L->refrac_count[k] - L->dt;
            v = v + xin;
            int s = v >= par(L, SNN_PN_THRESH, L->thresh, j);                        /* :519 */
            if (s) { rc = L->refrac; v = L->reset; }
            if (L->has_lbound && v < L->lbound) v = L->lbound;
            L->v[k] = v; L->refrac_count[k] = rc; L->s[k] = (uint8_t)s;
            pn_trace_and_sum(L, k, j, s, xin);
        }
    } else {
        uint8_t *cand = ws->cand;
        if (L->learning)
            for (int j = 0; j < n; ++j) L->theta[j] = L->theta[j] * par(L, SNN_PN_THETA_DECAY, L->theta_decay, j); /* :1078-1079 */
        for (size_t k = 0; k < BN; ++k) {
            const int j = (int)(k % (size_t)n);
            const float rest = par(L, SNN_PN_REST, L->rest, j);
            float v = par(L, SNN_PN_DECAY, L->decay, j) * (L->v[k] - rest) + rest;   /* :1077 */
            const float gate = L->refrac_count[k] <= 0.0f ? 1.0f : 0.0f;
            v = v + gate * cur[k];
            float rc = L->refrac_count[k] - L->dt;
            int s = v >= (par(L, SNN_PN_THRESH, L->thresh, j) + L->theta[j]);        /* :1088 */
            if (s) { rc = L->refrac; v = L->reset; }
            L->v[k] = v; L->refrac_count[k] = rc; cand[k] = (uint8_t)s;
        }
        if (L->learning)
            for (int j = 0; j < n; ++j) {
                int cnt = 0;
                for (int b = 0; b < B; ++b) cnt += cand[(size_t)b * n + j];
                L->theta[j] = L->theta[j] + par(L, SNN_PN_THETA_PLUS, L->theta_plus, j) * (float)cnt; /* :1093-1094 */
            }
        for (int b = 0; b < B; ++b) {
            uint8_t *cb = cand + (size_t)b * n;
            uint8_t *sb = L->s + (size_t)b * n;
            if (L->one_spike) {
                uint64_t best = 0;
                for (int j = 0; j < n; ++j)
                    if (cb[j]) {
                        uint64_t key = snn_one_spike_key(o->seed, (uint32_t)t + o->step_offset, (uint32_t)l, (uint32_t)b, (uint32_t)j);
                        if (key > best) best = key;
                    }
                for (int j = 0; j < n; ++j) sb[j] = 0;
                if (best) sb[(uint32_t)(best & 0xFFFFFFFFu)] = 1;
            } else {
                for (int j = 0; j < n; ++j) sb[j] = cb[j];
            }
        }
        for (size_t k = 0; k < BN; ++k) {
            if (L->has_lbound && L->v[k] < L->lbound) L->v[k] = L->lbound;
            pn_trace_and_sum(L, k, (int)(k % (size_t)n), L->s[k], cur[k]);
        }
    }
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

int snn_oracle_conn_update(const snn_net_t *net, int32_t ci, int32_t B) { return syn_conn_update_entry(net, ci, B); }

/* Network.run (network.py:252-465): the synapse-tensor oracle's timestep loop, with the step above for the layers that
 * carry a per-neuron block. */
int snn_oracle_run_window(const snn_net_t *net, const snn_run_opts_t *o, int dense, int threads) {
    static snn_net_t P;   /* the plan with the flags stripped (large for the stack; one window at a time) */
    if (!net || !o || net->n_layers < 1 || net->n_layers > SNN_MAX_LAYERS) return SNN_ERR_BAD_ARG;
    int any = 0;
    uint8_t pn[SNN_MAX_LAYERS] = {0};
    memcpy(&P, net, sizeof(P));
    for (int l = 0; l < net->n_layers; ++l) {
        snn_layer_t *L = &P.layers[l];
        if (!(L->kind & SNN_NODE_PN)) continue;
        const int rc = pn_check(L);
        if (rc) return rc;
        L->kind &= ~SNN_NODE_PN;
        pn[l] = L->pn_mask != 0u;
        any |= pn[l];
    }
    if (!any) return syn_run_window(&P, o, dense, threads);
    net = &P;
    for (int c = 0; c < net->n_conns && c < SNN_MAX_CONNS; ++c)
        if (has_syn(&net->conns[c])) {
            const int rc = syn_check(&net->conns[c]);
            if (rc) return rc;
        }
    int rc = check_plan(net, o);
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
        for (int l = 0; l < net->n_layers; ++l) lws[l].has_in = 0;
        for (int c = 0; c < net->n_conns && !o->one_step; ++c) {
            const snn_conn_t *C = &net->conns[c];
            const snn_layer_t *G = &net->layers[C->tgt];
            if (!lws[C->tgt].has_in) { memset(lws[C->tgt].cur, 0, sizeof(float) * (size_t)B * G->n); lws[C->tgt].has_in = 1; }
            if (C->kind == SNN_CONN_CONV2D) conv_compute(C, &net->layers[C->src], B, lws[C->tgt].cur, dense);
            else conn_compute(C, &net->layers[C->src], G->n, B, lws[C->tgt].cur, dense);
        }
        for (int l = 0; l < net->n_layers; ++l) {
            if (o->one_step)
                for (int c = 0; c < net->n_conns; ++c) {
                    const snn_conn_t *C = &net->conns[c];
                    if (C->tgt != l) continue;
                    const snn_layer_t *G = &net->layers[l];
                    if (!lws[l].has_in) { memset(lws[l].cur, 0, sizeof(float) * (size_t)B * G->n); lws[l].has_in = 1; }
                    if (C->kind == SNN_CONN_CONV2D) conv_compute(C, &net->layers[C->src], B, lws[l].cur, dense);
                    else conn_compute(C, &net->layers[C->src], G->n, B, lws[l].cur, dense);
                }
            if (pn[l]) pn_layer_forward(net, l, o, t, &lws[l]);
            else layer_forward(net, l, o, t, &lws[l], &err);
        }
        if (net->learning)
            for (int c = 0; c < net->n_conns; ++c) {
                const snn_conn_t *C = &net->conns[c];
                if (has_syn(C) && SNN_RULE_IS_MSTDP(C->rule)) syn_mstdp_update(net, C, o, dense);
                else if (has_syn(C)) syn_conn_update(net, C, o, &cws[c], dense);
                else if (C->rule == SNN_RULE_MSTDP && C->kind == SNN_CONN_CONV2D) mstdp_conv_update(net, C, o, dense);
                else if (C->rule == SNN_RULE_MSTDP) mstdp_dense_update(net, C, o, dense);
                else if (C->rule == SNN_RULE_MSTDPET) mstdpet_dense_update(net, C);
                else if (C->kind == SNN_CONN_CONV2D && SNN_RULE_IS_STDP(C->rule)) stdp_conv_update(net, C, o, dense);
                else if (C->kind == SNN_CONN_CONV2D) {
                    if (C->rule == SNN_RULE_NOOP && C->weight_decay != 0.0f)
                        for (size_t k = 0; k < (size_t)C->cout * C->cin * C->kh * C->kw; ++k) C->w[k] = C->w[k] * C->weight_decay;
                } else conn_update(net, C, o, &cws[c], dense);
            }
        for (int c = 0; c < net->n_conns; ++c) {
            const snn_conn_t *C = &net->conns[c];
            if (!C->mask || C->kind != SNN_CONN_DENSE) continue;
            const size_t NW = (size_t)net->layers[C->src].n * net->layers[C->tgt].n;
            for (size_t k = 0; k < NW; ++k) if (C->mask[k]) C->w[k] = 0.0f;
        }
        for (int l = 0; l < net->n_layers; ++l) {
            const snn_layer_t *L = &net->layers[l];
            const size_t BN = (size_t)B * L->n;
            if (L->rec_s) memcpy(L->rec_s + (size_t)t * BN, L->s, BN);
            if (L->rec_v && L->v) memcpy(L->rec_v + (size_t)t * BN, L->v, BN * sizeof(float));
            if (L->rec_count) for (size_t k = 0; k < BN; ++k) L->rec_count[k] += L->s[k] ? 1 : 0;
        }
    }
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
