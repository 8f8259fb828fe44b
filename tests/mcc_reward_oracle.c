/*
 * mcc_reward_oracle.c — TEST INFRASTRUCTURE: the feature oracle (tests/feature_oracle.c, which includes the CPU oracle
 * oracle/snn_oracle.c; both included unchanged) extended by the reward-modulated rules MCC_learning.MSTDP and
 * MCC_learning.MSTDPET on a MulticompartmentConnection's Weight (SNN_RULE_MSTDP / SNN_RULE_MSTDPET on SNN_CONN_MCC).  It
 * exports the oracle's own entry points, so it is a drop-in superset of libsnn_feature_oracle.so: plans without such a
 * rule go to the feature oracle's window untouched.
 *
 * MCC_learning.MSTDP._connection_update (MCC_learning.py:468-548) and MSTDPET._connection_update (:652-733) are, op for
 * op, learning.MSTDP._connection_update (learning.py:1504-1574) and learning.MSTDPET._connection_update (:2187-2249) with
 * the Weight's value in place of w and the rule's range in place of [wmin, wmax]; the base update (MCC_learning.py:86-110)
 * is learning.py:87-104's decay then clamp.  So the oracle's mstdp_dense_update / mstdpet_dense_update are the update,
 * and the plan is checked as the oracle checks the dense rule.  The rules read the Weight and the spikes only: a
 * Probability draw or a Mask changes what a synapse transmits, not what it learns.
 *
 *   gcc -O2 -fPIC -std=c11 -ffp-contract=off -fno-fast-math -fopenmp -shared -o libsnn_mcc_reward_oracle.so mcc_reward_oracle.c -lm
 */
#include "../include/snn_b200.h"

/* The feature oracle's window keeps its code but not its symbol: this declaration gives it another assembler name, and
 * the window below takes the exported one. */
int snn_oracle_run_window(const snn_net_t *net, const snn_run_opts_t *o, int dense, int threads) __asm__("feature_oracle_run_window");
#include "feature_oracle.c"

int mcc_reward_run_window(const snn_net_t *net, const snn_run_opts_t *o, int dense, int threads) __asm__("snn_oracle_run_window");

static int is_mcc_reward(const snn_conn_t *C) { return C->kind == SNN_CONN_MCC && SNN_RULE_IS_MSTDP(C->rule); }

/* check_plan with each MCC reward rule checked as the oracle checks the same rule on a dense Connection (the same fields
 * and pointers), and features only on MulticompartmentConnections. */
static int reward_check_plan(const snn_net_t *net, const snn_run_opts_t *o) {
    static snn_net_t as_dense;   /* large for the stack; the oracle runs one window at a time */
    memcpy(&as_dense, net, sizeof(as_dense));
    for (int c = 0; c < net->n_conns; ++c) {
        if (has_features(&net->conns[c]) && net->conns[c].kind != SNN_CONN_MCC) return SNN_ERR_BAD_ARG;
        if (is_mcc_reward(&net->conns[c])) as_dense.conns[c].kind = SNN_CONN_DENSE;
    }
    return check_plan(&as_dense, o);
}

/* Network.run (network.py:252-465): tests/feature_oracle.c's timestep loop, whose learning phase already applies
 * mstdp_dense_update / mstdpet_dense_update to every non-convolutional connection with such a rule. */
int mcc_reward_run_window(const snn_net_t *net, const snn_run_opts_t *o, int dense, int threads) {
    if (!net || !o) return SNN_ERR_BAD_ARG;
    int any = 0;
    for (int c = 0; c < net->n_conns && c < SNN_MAX_CONNS; ++c) any |= is_mcc_reward(&net->conns[c]);
    if (!any) return snn_oracle_run_window(net, o, dense, threads);
    int rc = reward_check_plan(net, o);
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
        /* 3. connection updates in insertion order (network.py:431-454; MulticompartmentConnection.update,
         *    topology.py:509-518: the Weight's rule) */
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
