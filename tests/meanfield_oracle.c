/*
 * meanfield_oracle.c — TEST INFRASTRUCTURE: the CPU oracle (oracle/snn_oracle.c, included unchanged) extended by
 * MeanFieldConnection (SNN_CONN_MEANFIELD).  It exports the oracle's entry points as they are, and its own window and
 * compute under the names snn_oracle_mf_*, which tests/meanfield_oracle.py puts in the place of the oracle's: plans
 * without a mean-field connection go to the oracle's functions untouched.
 *
 * MeanFieldConnection.compute (topology.py:1972-1981), called once per step by _get_inputs (network.py:244-248) on the
 * source's current spikes s [B, n_src]:
 *   s.float().mean() * w         the mean over the whole tensor, the batch included
 * The CPU sum of B * n_src values 0.0 / 1.0 is the integer spike count (exact below 2^24), and the mean is that sum
 * divided by float(B * n_src), one rounding; the product with each element of w is one more.  network.py:248 then adds
 * the broadcast result into the target's input, one rounding per element, in insertion order.  Here the broadcast is
 * spelled out through the plan's offset map: target j of sample b reads w[mf_off[j] + b * mf_stride].
 * learning.NoOp scales w by 1.0 and never clamps (learning.py:93-104): w is not touched.
 *
 *   gcc -O2 -fPIC -std=c11 -ffp-contract=off -fno-fast-math -fopenmp -shared -o libsnn_meanfield_oracle.so meanfield_oracle.c -lm
 */
#include "../oracle/snn_oracle.c"

/* include/snn_b200.h's conditions on a mean-field connection. */
static int mf_check(const snn_conn_t *C, int n_src, int B) {
    if (!C->w || !C->mf_off || C->b || C->mf_stride < 0 || (long long)B * n_src >= (1LL << 24)) return SNN_ERR_BAD_ARG;
    if ((C->rule != SNN_RULE_NONE && C->rule != SNN_RULE_NOOP) || C->has_norm || C->mask) return SNN_ERR_UNSUPPORTED;
    return SNN_OK;
}

/* One compute call on spikes s [B, n_src], added into cur [B, n_tgt] like network.py:248 (add = 0: stored, as the
 * standalone compute returns it). */
static void mf_compute(const snn_conn_t *C, const uint8_t *s, int n_src, int n_tgt, int B, float *cur, int add) {
    const size_t N = (size_t)B * n_src;
    float sum = 0.0f;   /* torch's float sum of 0.0 / 1.0 values: the count, exactly */
    for (size_t k = 0; k < N; ++k) sum = sum + (s[k] ? 1.0f : 0.0f);
    const float mean = sum / (float)N;
    for (int b = 0; b < B; ++b)
        for (int j = 0; j < n_tgt; ++j) {
            const float p = mean * C->w[C->mf_off[j] + (size_t)b * C->mf_stride];
            cur[(size_t)b * n_tgt + j] = add ? cur[(size_t)b * n_tgt + j] + p : p;
        }
}

static void any_mf_compute(const snn_net_t *net, int c, int B, float *cur, int dense) {
    const snn_conn_t *C = &net->conns[c];
    const snn_layer_t *S = &net->layers[C->src];
    const int nt = net->layers[C->tgt].n;
    if (C->kind == SNN_CONN_MEANFIELD) mf_compute(C, S->s, S->n, nt, B, cur, 1);
    else if (C->kind == SNN_CONN_CONV2D) conv_compute(C, S, B, cur, dense);
    else conn_compute(C, S, nt, B, cur, dense);
}

int snn_oracle_mf_run_window(const snn_net_t *net, const snn_run_opts_t *o, int dense, int threads);
int snn_oracle_mf_conn_compute(const snn_conn_t *C, int32_t n_src, int32_t n_tgt, int32_t B, const uint8_t *s, float *out);

/* Network.run (network.py:252-465): the oracle's timestep loop with the mean-field connection in _get_inputs. */
int snn_oracle_mf_run_window(const snn_net_t *net, const snn_run_opts_t *o, int dense, int threads) {
    if (!net || !o || net->n_conns < 0 || net->n_conns > SNN_MAX_CONNS || net->n_layers < 1 || net->n_layers > SNN_MAX_LAYERS) return SNN_ERR_BAD_ARG;
    int any = 0;
    for (int c = 0; c < net->n_conns; ++c) any |= net->conns[c].kind == SNN_CONN_MEANFIELD;
    if (!any) return snn_oracle_run_window(net, o, dense, threads);
    /* the oracle's own plan checks on everything but the mean-field connections, which are checked here */
    snn_net_t rest = *net;
    rest.n_conns = 0;
    for (int c = 0; c < net->n_conns; ++c) {
        const snn_conn_t *C = &net->conns[c];
        if (C->kind != SNN_CONN_MEANFIELD) { rest.conns[rest.n_conns++] = *C; continue; }
        if (C->src < 0 || C->src >= net->n_layers || C->tgt < 0 || C->tgt >= net->n_layers) return SNN_ERR_BAD_ARG;
        if (net->layers[C->tgt].kind == SNN_NODE_INPUT) return SNN_ERR_UNSUPPORTED;
        const int rc = mf_check(C, net->layers[C->src].n, o->B);
        if (rc) return rc;
    }
    int rc = check_plan(&rest, o);
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
            any_mf_compute(net, c, B, lws[C->tgt].cur, dense);
        }
        /* 2. layers in insertion order (network.py:386-429); one-step mode recomputes a layer's input just before it */
        for (int l = 0; l < net->n_layers; ++l) {
            if (o->one_step)
                for (int c = 0; c < net->n_conns; ++c) {
                    const snn_conn_t *C = &net->conns[c];
                    if (C->tgt != l) continue;
                    if (!lws[l].has_in) { memset(lws[l].cur, 0, sizeof(float) * (size_t)B * net->layers[l].n); lws[l].has_in = 1; }
                    any_mf_compute(net, c, B, lws[l].cur, dense);
                }
            layer_forward(net, l, o, t, &lws[l], &err);
        }
        /* 3. connection updates in insertion order (network.py:431-454); learning.NoOp leaves a mean-field w as it is */
        if (net->learning)
            for (int c = 0; c < net->n_conns; ++c) {
                const snn_conn_t *C = &net->conns[c];
                if (C->kind == SNN_CONN_MEANFIELD) continue;
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
    /* network.py:464-465; a mean-field connection has no norm */
    if (o->normalize)
        for (int c = 0; c < net->n_conns; ++c) {
            const snn_conn_t *C = &net->conns[c];
            if (C->kind == SNN_CONN_MEANFIELD || !C->has_norm) continue;
            if (C->kind == SNN_CONN_CONV2D) normalize_conv(C);
            else normalize_cols(C->w, net->layers[C->src].n, net->layers[C->tgt].n, C->norm_abs, C->norm);
        }
    for (int l = 0; l < net->n_layers; ++l) { free(lws[l].cur); free(lws[l].cand); }
    for (int c = 0; c < net->n_conns; ++c) { free(cws[c].U); free(cws[c].V); free(cws[c].tx); free(cws[c].row_t); free(cws[c].col_t); }
    if (o->err_flag) *o->err_flag |= err;
    return SNN_OK;
}

/* MeanFieldConnection.compute: out [B, n_tgt] = fl(mean * w[...]), the values the window adds into the input. */
int snn_oracle_mf_conn_compute(const snn_conn_t *C, int32_t n_src, int32_t n_tgt, int32_t B, const uint8_t *s, float *out) {
    if (!C || C->kind != SNN_CONN_MEANFIELD) return snn_oracle_conn_compute(C, n_src, n_tgt, B, s, out);
    if (!s || !out || B <= 0 || n_src <= 0 || n_tgt <= 0) return SNN_ERR_BAD_ARG;
    const int rc = mf_check(C, n_src, B);
    if (rc) return rc;
    mf_compute(C, s, n_src, n_tgt, B, out, 0);
    return SNN_OK;
}
