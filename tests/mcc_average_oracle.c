/*
 * mcc_average_oracle.c — TEST INFRASTRUCTURE: the feature oracle (tests/feature_oracle.c, which includes the CPU oracle
 * oracle/snn_oracle.c; both included unchanged) extended by MCC_learning.PostPre with average_update (SNN_RULE_MCC_POSTPRE
 * | SNN_RULE_AVG, include/snn_b200.h).  It exports the oracle's own entry points, so it is a drop-in superset of
 * libsnn_feature_oracle.so: plans without an averaged rule go to the feature oracle's window and single-operator update
 * untouched.
 *
 * PostPre._connection_update (MCC_learning.py:224-302) with average_update = k: each side whose rate is non-zero writes
 * its step's batch-reduced term (no dt) into slot `index` of its buffer, advances the index mod k, and — every update
 * with continues_update, else when the index wrapped to 0 — applies mean(buffer, 0) * dt to the Weight (pre: -=,
 * post: +=); then decay and clamp (:86-110).  The order is fixed as the header states: the mean of an element is its
 * slots summed in ascending order from +0, divided by k, times dt.  Slots outside a side's recorded rows / columns
 * hold zeros and are skipped, which leaves such a sum as it is, and an element no slot covers keeps its value.
 *
 *   gcc -O2 -fPIC -std=c11 -ffp-contract=off -fno-fast-math -fopenmp -shared -o libsnn_mcc_average_oracle.so mcc_average_oracle.c -lm
 */
#include "../include/snn_b200.h"

/* The feature oracle's window and single-operator update keep their code but not their symbols: these declarations
 * give them other assembler names, and the functions below take the exported ones. */
int snn_oracle_run_window(const snn_net_t *net, const snn_run_opts_t *o, int dense, int threads) __asm__("feature_oracle_run_window");
int snn_oracle_conn_update(const snn_net_t *net, int32_t ci, int32_t B) __asm__("feature_oracle_conn_update");
#include "feature_oracle.c"

int mcc_average_run_window(const snn_net_t *net, const snn_run_opts_t *o, int dense, int threads) __asm__("snn_oracle_run_window");
int mcc_average_conn_update(const snn_net_t *net, int32_t ci, int32_t B) __asm__("snn_oracle_conn_update");

static int is_avg(const snn_conn_t *C) { return (C->rule & SNN_RULE_AVG) != 0; }

static int avg_fields_ok(const snn_conn_t *C) {
    if ((C->rule & ~SNN_RULE_AVG) != SNN_RULE_MCC_POSTPRE || C->kind != SNN_CONN_MCC || C->mask) return SNN_ERR_UNSUPPORTED;
    if (C->avg_k < 1 || C->avg_idx_pre < 0 || C->avg_idx_pre >= C->avg_k || C->avg_idx_post < 0 || C->avg_idx_post >= C->avg_k)
        return SNN_ERR_BAD_ARG;
    if (!C->avg_pre || !C->avg_post || !C->avg_rows || !C->avg_cols) return SNN_ERR_BAD_ARG;
    return SNN_OK;
}

/* check_plan with every averaged rule checked as the plain MCC PostPre, and features only on MulticompartmentConnections */
static int average_check_plan(const snn_net_t *net, const snn_run_opts_t *o) {
    static snn_net_t plain;   /* large for the stack; the oracle runs one window at a time */
    memcpy(&plain, net, sizeof(plain));
    for (int c = 0; c < net->n_conns; ++c) {
        if (has_features(&net->conns[c]) && net->conns[c].kind != SNN_CONN_MCC) return SNN_ERR_BAD_ARG;
        if (is_avg(&net->conns[c])) {
            const int rc = avg_fields_ok(&net->conns[c]);
            if (rc) return rc;
            plain.conns[c].rule = SNN_RULE_MCC_POSTPRE;
        }
    }
    return check_plan(&plain, o);
}

static int bit(const uint32_t *words, int i) { return (words[i >> 5] >> (i & 31)) & 1u; }

/* One update of an averaged MCC PostPre from the layers' current s / x; `step` = updates of this rule already made since
 * the plan's indices (the window's step t). */
static void avg_update(const snn_net_t *net, const snn_conn_t *C, int B, int step, int first) {
    const snn_layer_t *S = &net->layers[C->src], *G = &net->layers[C->tgt];
    const int ns = S->n, nt = G->n, K = C->avg_k, nwS = (ns + 31) / 32, nwG = (nt + 31) / 32;
    const size_t KS = (size_t)ns * nt;
    const float Bf = (float)B, Kf = (float)K;
    const int pre_on = C->nu0 != 0.0f, post_on = C->nu1 != 0.0f;
    const int pp = (C->avg_idx_pre + step) % K, pq = (C->avg_idx_post + step) % K;
    const int apply_pre = pre_on && (C->avg_continues || (pp + 1) % K == 0);
    const int apply_post = post_on && (C->avg_continues || (pq + 1) % K == 0);
    uint8_t *pre_hit = (uint8_t *)calloc((size_t)ns, 1), *post_hit = (uint8_t *)calloc((size_t)nt, 1);
    if (pre_on) {
        /* slot pp = reduce_b s_src[b,i] * (x_tgt[b,j] * nu0) on the rows with a spike now, zeros where the previous occupant
         * had some; samples ascending from +0 */
        uint32_t *rows = C->avg_rows + (size_t)pp * nwS;
        float *slot = C->avg_pre + (size_t)pp * KS;
#pragma omp parallel for schedule(static)
        for (int i = 0; i < ns; ++i) {
            int now = 0;
            for (int b = 0; b < B; ++b) now |= S->s[(size_t)b * ns + i] != 0;
            if (!now && !bit(rows, i)) continue;
            float *row = slot + (size_t)i * nt;
            for (int j = 0; j < nt; ++j) row[j] = 0.0f;
            for (int b = 0; b < B; ++b)   /* each element's samples ascending */
                if (S->s[(size_t)b * ns + i])
                    for (int j = 0; j < nt; ++j) row[j] = row[j] + G->x[(size_t)b * nt + j] * C->nu0;
            if (now && C->reduction == SNN_REDUCE_MEAN) for (int j = 0; j < nt; ++j) row[j] = row[j] / Bf;
        }
        for (int i = 0; i < ns; ++i) {
            int now = 0;
            for (int b = 0; b < B; ++b) now |= S->s[(size_t)b * ns + i] != 0;
            if (now) rows[i >> 5] |= 1u << (i & 31);
            else rows[i >> 5] &= ~(1u << (i & 31));
        }
        if (apply_pre) {
#pragma omp parallel for schedule(static)
            for (int i = 0; i < ns; ++i) {
                int any = 0;
                for (int q = 0; q < K; ++q) any |= bit(C->avg_rows + (size_t)q * nwS, i);
                if (!any) continue;
                pre_hit[i] = 1;
                float *acc = (float *)calloc((size_t)nt, sizeof(float));   /* each element's slots ascending from +0 */
                for (int q = 0; q < K; ++q)
                    if (bit(C->avg_rows + (size_t)q * nwS, i))
                        for (int j = 0; j < nt; ++j) acc[j] = acc[j] + C->avg_pre[(size_t)q * KS + (size_t)i * nt + j];
                for (int j = 0; j < nt; ++j) {
                    float d = acc[j] / Kf;
                    d = d * C->dt_scale;
                    C->w[(size_t)i * nt + j] = C->w[(size_t)i * nt + j] - d;
                }
                free(acc);
            }
        }
    }
    if (post_on) {
        /* slot pq = reduce_b x_src[b,i] * (s_tgt[b,j] * nu1) on the columns with a spike now */
        uint32_t *cols = C->avg_cols + (size_t)pq * nwG;
        float *slot = C->avg_post + (size_t)pq * KS;
        for (int j = 0; j < nt; ++j) {
            int now = 0;
            for (int b = 0; b < B; ++b) now |= G->s[(size_t)b * nt + j] != 0;
            if (!now && !bit(cols, j)) continue;
            for (int i = 0; i < ns; ++i) slot[(size_t)i * nt + j] = 0.0f;
            for (int b = 0; b < B; ++b)   /* each element's samples ascending */
                if (G->s[(size_t)b * nt + j])
                    for (int i = 0; i < ns; ++i) slot[(size_t)i * nt + j] = slot[(size_t)i * nt + j] + S->x[(size_t)b * ns + i] * C->nu1;
            if (now && C->reduction == SNN_REDUCE_MEAN) for (int i = 0; i < ns; ++i) slot[(size_t)i * nt + j] = slot[(size_t)i * nt + j] / Bf;
            if (now) cols[j >> 5] |= 1u << (j & 31);
            else cols[j >> 5] &= ~(1u << (j & 31));
        }
        if (apply_post)
#pragma omp parallel for schedule(static)
            for (int j = 0; j < nt; ++j) {
                int any = 0;
                for (int q = 0; q < K; ++q) any |= bit(C->avg_cols + (size_t)q * nwG, j);
                if (!any) continue;
                post_hit[j] = 1;
                for (int i = 0; i < ns; ++i) {
                    float s = 0.0f;
                    for (int q = 0; q < K; ++q)
                        if (bit(C->avg_cols + (size_t)q * nwG, j)) s = s + C->avg_post[(size_t)q * KS + (size_t)i * nt + j];
                    float d = s / Kf;
                    d = d * C->dt_scale;
                    C->w[(size_t)i * nt + j] = C->w[(size_t)i * nt + j] + d;
                }
            }
    }
    /* decay and clamp (MCC_learning.py:86-110) on every element the terms reached; every element when the decay is on or
     * at the first update (entries may lie outside the range) — elsewhere both are bitwise no-ops */
    const int full = (C->weight_decay != 0.0f && C->weight_decay != 1.0f) || (C->has_clamp && first);
#pragma omp parallel for schedule(static)
    for (int i = 0; i < ns; ++i)
        for (int j = 0; j < nt; ++j) {
            if (!full && !pre_hit[i] && !post_hit[j]) continue;
            float w = C->w[(size_t)i * nt + j];
            if (C->weight_decay != 0.0f) w = w * C->weight_decay;
            if (C->has_clamp) w = w < C->wmin ? C->wmin : (w > C->wmax ? C->wmax : w);
            C->w[(size_t)i * nt + j] = w;
        }
    free(pre_hit); free(post_hit);
}

/* Network.run (network.py:252-465): tests/feature_oracle.c's timestep loop, as tests/mcc_reward_oracle.c runs it, with
 * the averaged rules updated by avg_update. */
int mcc_average_run_window(const snn_net_t *net, const snn_run_opts_t *o, int dense, int threads) {
    if (!net || !o) return SNN_ERR_BAD_ARG;
    int any = 0;
    for (int c = 0; c < net->n_conns && c < SNN_MAX_CONNS; ++c) any |= is_avg(&net->conns[c]);
    if (!any) return snn_oracle_run_window(net, o, dense, threads);
    int rc = average_check_plan(net, o);
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
        }
        /* 2. layers in insertion order (network.py:386-429); one-step mode recomputes a layer's input just before it */
        for (int l = 0; l < net->n_layers; ++l) {
            if (o->one_step)
                for (int c = 0; c < net->n_conns; ++c) {
                    const snn_conn_t *C = &net->conns[c];
                    if (C->tgt != l) continue;
                    if (!lws[l].has_in) { memset(lws[l].cur, 0, sizeof(float) * (size_t)B * net->layers[l].n); lws[l].has_in = 1; }
                    any_compute(net, c, o, t, lws[l].cur, dense);
                }
            layer_forward(net, l, o, t, &lws[l], &err);
        }
        /* 3. connection updates in insertion order (network.py:431-454) */
        if (net->learning)
            for (int c = 0; c < net->n_conns; ++c) {
                const snn_conn_t *C = &net->conns[c];
                if (is_avg(C)) avg_update(net, C, B, t, t == 0);
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
    /* network.py:464-465 */
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

/* connection.update(learning=True) (MCC_learning.py:224-302) for an averaged rule; any other goes to the feature oracle */
int mcc_average_conn_update(const snn_net_t *net, int32_t ci, int32_t B) {
    if (!net || ci < 0 || ci >= net->n_conns) return SNN_ERR_BAD_ARG;
    const snn_conn_t *C = &net->conns[ci];
    if (!is_avg(C)) return snn_oracle_conn_update(net, ci, B);
    const int rc = avg_fields_ok(C);
    if (rc) return rc;
    avg_update(net, C, B, 0, 1);
    return SNN_OK;
}
