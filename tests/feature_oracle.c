/*
 * feature_oracle.c — TEST INFRASTRUCTURE: the CPU oracle (oracle/snn_oracle.c, included unchanged) extended by the
 * MulticompartmentConnection features Probability, Mask and Intensity (snn_conn_t f_prob / f_mask / f_int).  It
 * exports the oracle's own entry points, so it is a drop-in superset of libsnn_oracle.so: plans without a feature go
 * to the oracle's functions untouched.  The oracle itself stays byte for byte what every other test compares with;
 * the features are restated here, as tests/sparse_oracle.c restates the sparse kind.
 *
 * MulticompartmentConnection.compute (topology.py:437-479) broadcasts the spikes to [B, n_src, n_tgt], multiplies the
 * broadcast by each feature of the pipeline in turn and sums over the sources (:471):
 *   Probability  conn_spikes * torch.bernoulli(value)   topology_features.py:425-429 — one [n_src, n_tgt] draw per
 *                call, shared by the batch; drawn here with snn_synapse_draw (include/snn_b200.h), as the golden
 *                generator patches the reference to do
 *   Mask         conn_spikes * value                    :507-508
 *   Intensity    conn_spikes * value                    :755-756
 *   Weight       value * conn_spikes                    :641
 * The spike and the Probability / Mask factors are exact 0 / 1, so each product is 0 or the one rounding of w * I,
 * whatever the pipeline order.  Same arithmetic contract as the oracle (-ffp-contract=off, one rounding per
 * reference op); `dense` = 1 evaluates every product of the broadcast, zeros included.
 *
 *   gcc -O2 -fPIC -std=c11 -ffp-contract=off -fno-fast-math -fopenmp -shared -o libsnn_feature_oracle.so feature_oracle.c -lm
 */
#define snn_oracle_run_window oracle_run_window_base
#define snn_oracle_conn_compute oracle_conn_compute_base
#include "../oracle/snn_oracle.c"
#undef snn_oracle_run_window
#undef snn_oracle_conn_compute

int snn_oracle_run_window(const snn_net_t *net, const snn_run_opts_t *o, int dense, int threads);
int snn_oracle_conn_compute(const snn_conn_t *C, int32_t n_src, int32_t n_tgt, int32_t B, const uint8_t *s, float *out);

static int has_features(const snn_conn_t *C) { return C->f_prob || C->f_mask || C->f_int; }

/* The pipeline's product for every synapse of a step, added into the target's accumulator like network.py:248. */
static void feature_compute(const snn_conn_t *C, const snn_layer_t *S, int n_tgt, int B, float *cur, int dense, uint32_t seed,
                            uint32_t step, uint32_t conn) {
    const int ns = S->n;
    const size_t NW = (size_t)ns * n_tgt;
    float *bern = NULL;   /* torch.bernoulli(value): one draw for the whole batch */
    if (C->f_prob) {
        bern = (float *)malloc(sizeof(float) * NW);
#pragma omp parallel for schedule(static)
        for (int i = 0; i < ns; ++i)
            for (int j = 0; j < n_tgt; ++j) {
                const size_t ij = (size_t)i * n_tgt + j;
                bern[ij] = snn_synapse_transmits(snn_synapse_draw(seed, step, conn, (uint32_t)i, (uint32_t)j), C->f_prob[ij]) ? 1.0f : 0.0f;
            }
    }
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
                for (int j = 0; j < n_tgt; ++j) {
                    const size_t ij = (size_t)i * n_tgt + j;
                    float x = sv;
                    if (bern) x = x * bern[ij];
                    if (C->f_mask) x = x * (C->f_mask[ij] ? 1.0f : 0.0f);
                    if (!dense && x == 0.0f) continue;   /* a dropped synapse adds nothing */
                    if (C->f_int) x = x * C->f_int[ij];
                    p[j] = p[j] + C->w[ij] * x;
                }
            }
            float *cb = cur + (size_t)b * n_tgt;
            for (int j = 0; j < n_tgt; ++j) cb[j] = cb[j] + p[j];
        }
        free(p);
    }
    free(bern);
}

static void any_compute(const snn_net_t *net, int c, const snn_run_opts_t *o, int t, float *cur, int dense) {
    const snn_conn_t *C = &net->conns[c];
    const snn_layer_t *S = &net->layers[C->src];
    const int nt = net->layers[C->tgt].n;
    if (C->kind == SNN_CONN_CONV2D) conv_compute(C, S, o->B, cur, dense);
    else if (has_features(C)) feature_compute(C, S, nt, o->B, cur, dense, o->seed, o->step_offset + (uint32_t)t, (uint32_t)c);
    else conn_compute(C, S, nt, o->B, cur, dense);
}

/* Network.run (network.py:252-465): oracle/snn_oracle.c's timestep loop with the feature pipeline in _get_inputs. */
int snn_oracle_run_window(const snn_net_t *net, const snn_run_opts_t *o, int dense, int threads) {
    if (!net || !o) return SNN_ERR_BAD_ARG;
    int any = 0;
    for (int c = 0; c < net->n_conns && c < SNN_MAX_CONNS; ++c) {
        if (has_features(&net->conns[c]) && net->conns[c].kind != SNN_CONN_MCC) return SNN_ERR_BAD_ARG;
        any |= has_features(&net->conns[c]);
    }
    if (!any) return oracle_run_window_base(net, o, dense, threads);
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
    /* network.py:464-465: Weight.normalize (topology_features.py:250-266) reads the Weight only */
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

/* MulticompartmentConnection.compute with features, drawn under (draw_seed, draw_step, draw_conn). */
int snn_oracle_conn_compute(const snn_conn_t *C, int32_t n_src, int32_t n_tgt, int32_t B, const uint8_t *s, float *out) {
    if (!C || !has_features(C)) return oracle_conn_compute_base(C, n_src, n_tgt, B, s, out);
    if (C->kind != SNN_CONN_MCC || !C->w || !s || !out) return SNN_ERR_BAD_ARG;
    snn_layer_t S; memset(&S, 0, sizeof(S)); S.n = n_src; S.s = (uint8_t *)s;
    memset(out, 0, sizeof(float) * (size_t)B * n_tgt);
    feature_compute(C, &S, n_tgt, B, out, 0, C->draw_seed, C->draw_step, C->draw_conn);
    return SNN_OK;
}
