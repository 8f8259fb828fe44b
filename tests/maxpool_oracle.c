/*
 * maxpool_oracle.c — TEST INFRASTRUCTURE: the CPU oracle (oracle/snn_oracle.c, included unchanged) extended by
 * MaxPool2dConnection (SNN_CONN_MAXPOOL2D).  It exports the oracle's own entry points, so it is a drop-in superset of
 * libsnn_oracle.so: plans without a pooling connection go to the oracle's functions untouched.  The oracle itself stays
 * byte for byte what every other test compares with; the pooling connection is restated here, as tests/sparse_oracle.c
 * restates the sparse kind.
 *
 * MaxPool2dConnection.compute (topology.py:1163-1185), called once per step by _get_inputs (network.py:248) on the
 * source's current spikes:
 *   firing_rates -= decay * firing_rates           one rounding for the product, one for the difference
 *   firing_rates += s.float().squeeze()            one rounding
 *   _, idx = F.max_pool2d(firing_rates, ..., return_indices=True)
 *   out = s.flatten(2).gather(2, idx.flatten(2))   the spike at the window's first maximum
 * F.max_pool2d's CPU kernel scans the window's valid elements in row-major order and keeps the first one unless a later
 * one compares strictly greater (or is a NaN).  Same arithmetic contract as the oracle (-ffp-contract=off).
 *
 *   gcc -O2 -fPIC -std=c11 -ffp-contract=off -fno-fast-math -fopenmp -shared -o libsnn_maxpool_oracle.so maxpool_oracle.c -lm
 */
#define snn_oracle_run_window oracle_run_window_base
#define snn_oracle_conn_compute oracle_conn_compute_base
#include "../oracle/snn_oracle.c"
#undef snn_oracle_run_window
#undef snn_oracle_conn_compute

int snn_oracle_run_window(const snn_net_t *net, const snn_run_opts_t *o, int dense, int threads);
int snn_oracle_conn_compute(const snn_conn_t *C, int32_t n_src, int32_t n_tgt, int32_t B, const uint8_t *s, float *out);

/* include/snn_b200.h's conditions on a pooling connection: no weights, learning.NoOp, the F.max_pool2d geometry with a
 * valid element in every window. */
static int pool_check(const snn_conn_t *C, int n_src, int n_tgt) {
    if (C->w || C->b || !C->pool_rates) return SNN_ERR_BAD_ARG;
    if (C->rule != SNN_RULE_NOOP || C->has_norm || C->mask) return SNN_ERR_UNSUPPORTED;
    if (C->cin != C->cout || C->cin < 1 || C->cin * C->hin * C->win != n_src || C->cout * C->hout * C->wout != n_tgt) return SNN_ERR_BAD_ARG;
    if (C->kh < 1 || C->kw < 1 || C->sh < 1 || C->sw < 1 || C->dh < 1 || C->dw < 1 || C->ph < 0 || C->pw < 0) return SNN_ERR_BAD_ARG;
    if (C->ph > C->kh / 2 || C->pw > C->kw / 2) return SNN_ERR_BAD_ARG;
    const int eh = C->hin + 2 * C->ph - C->dh * (C->kh - 1) - 1, ew = C->win + 2 * C->pw - C->dw * (C->kw - 1) - 1;
    if (eh < 0 || ew < 0 || C->hout != eh / C->sh + 1 || C->wout != ew / C->sw + 1) return SNN_ERR_BAD_ARG;
    return SNN_OK;
}

/* One compute call: the rates of every sample advance by its spikes, then each target neuron takes the spike at its
 * window's first maximum; the result is added into `cur` like network.py:248. */
static void pool_compute(const snn_conn_t *C, const uint8_t *s, int B, float *cur) {
    const int HW = C->hin * C->win, ns = C->cin * HW, L = C->hout * C->wout, nt = C->cout * L;
#pragma omp parallel for schedule(static)
    for (int b = 0; b < B; ++b) {
        float *r = C->pool_rates + (size_t)b * ns;
        const uint8_t *sb = s + (size_t)b * ns;
        for (int i = 0; i < ns; ++i) {
            const float d = C->pool_decay * r[i];
            r[i] = r[i] - d;
            r[i] = r[i] + (sb[i] ? 1.0f : 0.0f);
        }
        for (int j = 0; j < nt; ++j) {
            const int ch = j / L, l = j - ch * L, oy = l / C->wout, ox = l - oy * C->wout;
            const float *rc = r + (size_t)ch * HW;
            float best = 0.0f;
            int idx = -1;
            for (int ky = 0; ky < C->kh; ++ky) {
                const int iy = oy * C->sh - C->ph + ky * C->dh;
                if (iy < 0 || iy >= C->hin) continue;
                for (int kx = 0; kx < C->kw; ++kx) {
                    const int ix = ox * C->sw - C->pw + kx * C->dw;
                    if (ix < 0 || ix >= C->win) continue;
                    const float v = rc[iy * C->win + ix];
                    if (idx < 0 || v > best || isnan(v)) { best = v; idx = iy * C->win + ix; }
                }
            }
            const float p = (idx >= 0 && sb[ch * HW + idx]) ? 1.0f : 0.0f;
            cur[(size_t)b * nt + j] = cur[(size_t)b * nt + j] + p;
        }
    }
}

static void any_compute(const snn_net_t *net, int c, const snn_run_opts_t *o, float *cur, int dense) {
    const snn_conn_t *C = &net->conns[c];
    const snn_layer_t *S = &net->layers[C->src];
    if (C->kind == SNN_CONN_MAXPOOL2D) pool_compute(C, S->s, o->B, cur);
    else if (C->kind == SNN_CONN_CONV2D) conv_compute(C, S, o->B, cur, dense);
    else conn_compute(C, S, net->layers[C->tgt].n, o->B, cur, dense);
}

/* Network.run (network.py:252-465): oracle/snn_oracle.c's timestep loop with the pooling connection in _get_inputs. */
int snn_oracle_run_window(const snn_net_t *net, const snn_run_opts_t *o, int dense, int threads) {
    if (!net || !o || net->n_conns < 0 || net->n_conns > SNN_MAX_CONNS || net->n_layers < 1 || net->n_layers > SNN_MAX_LAYERS) return SNN_ERR_BAD_ARG;
    int any = 0;
    for (int c = 0; c < net->n_conns; ++c) any |= net->conns[c].kind == SNN_CONN_MAXPOOL2D;
    if (!any) return oracle_run_window_base(net, o, dense, threads);
    /* the oracle's own plan checks on everything but the pooling connections, which are checked here */
    snn_net_t rest = *net;
    rest.n_conns = 0;
    for (int c = 0; c < net->n_conns; ++c) {
        const snn_conn_t *C = &net->conns[c];
        if (C->kind != SNN_CONN_MAXPOOL2D) { rest.conns[rest.n_conns++] = *C; continue; }
        if (C->src < 0 || C->src >= net->n_layers || C->tgt < 0 || C->tgt >= net->n_layers) return SNN_ERR_BAD_ARG;
        if (net->layers[C->tgt].kind == SNN_NODE_INPUT) return SNN_ERR_UNSUPPORTED;
        const int rc = pool_check(C, net->layers[C->src].n, net->layers[C->tgt].n);
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
            any_compute(net, c, o, lws[C->tgt].cur, dense);
        }
        /* 2. layers in insertion order (network.py:386-429); one-step mode recomputes a layer's input just before it */
        for (int l = 0; l < net->n_layers; ++l) {
            if (o->one_step)
                for (int c = 0; c < net->n_conns; ++c) {
                    const snn_conn_t *C = &net->conns[c];
                    if (C->tgt != l) continue;
                    if (!lws[l].has_in) { memset(lws[l].cur, 0, sizeof(float) * (size_t)B * net->layers[l].n); lws[l].has_in = 1; }
                    any_compute(net, c, o, lws[l].cur, dense);
                }
            layer_forward(net, l, o, t, &lws[l], &err);
        }
        /* 3. connection updates in insertion order (network.py:431-454); a pooling connection has nothing to update */
        if (net->learning)
            for (int c = 0; c < net->n_conns; ++c) {
                const snn_conn_t *C = &net->conns[c];
                if (C->kind == SNN_CONN_MAXPOOL2D) continue;
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
    /* network.py:464-465; MaxPool2dConnection.normalize does nothing (topology.py:1194-1199) */
    if (o->normalize)
        for (int c = 0; c < net->n_conns; ++c) {
            const snn_conn_t *C = &net->conns[c];
            if (C->kind == SNN_CONN_MAXPOOL2D || !C->has_norm) continue;
            if (C->kind == SNN_CONN_CONV2D) normalize_conv(C);
            else normalize_cols(C->w, net->layers[C->src].n, net->layers[C->tgt].n, C->norm_abs, C->norm);
        }
    for (int l = 0; l < net->n_layers; ++l) { free(lws[l].cur); free(lws[l].cand); }
    for (int c = 0; c < net->n_conns; ++c) { free(cws[c].U); free(cws[c].V); free(cws[c].tx); free(cws[c].row_t); free(cws[c].col_t); }
    if (o->err_flag) *o->err_flag |= err;
    return SNN_OK;
}

/* MaxPool2dConnection.compute: the rates in C->pool_rates advance in place, out is [B, C, hout, wout]. */
int snn_oracle_conn_compute(const snn_conn_t *C, int32_t n_src, int32_t n_tgt, int32_t B, const uint8_t *s, float *out) {
    if (!C || C->kind != SNN_CONN_MAXPOOL2D) return oracle_conn_compute_base(C, n_src, n_tgt, B, s, out);
    if (!s || !out || B <= 0) return SNN_ERR_BAD_ARG;
    const int rc = pool_check(C, n_src, n_tgt);
    if (rc) return rc;
    memset(out, 0, sizeof(float) * (size_t)B * n_tgt);
    pool_compute(C, s, B, out);
    return SNN_OK;
}
