/*
 * maxpool3d_oracle.c — TEST INFRASTRUCTURE: the CPU oracle extended by Conv3dConnection (tests/conv3d_oracle.c, which
 * includes oracle/snn_oracle.c; both included unchanged) and by MaxPoo3dConnection (SNN_CONN_MAXPOOL3D).  It exports
 * conv3d_oracle.c's entry points as they are, and its own window and compute under the names snn_oracle_mp3_*, which
 * tests/maxpool3d_oracle.py puts in the place of the oracle's: plans without a 3-D pooling connection go to
 * conv3d_oracle.c's functions untouched, and a Conv3d -> pool network runs here.
 *
 * MaxPoo3dConnection.compute (topology.py:1255-1277), called once per step by _get_inputs (network.py:248) on the
 * source's current spikes, source [C, din, hin, win], target [C, dout, hout, wout]:
 *   firing_rates -= decay * firing_rates           one rounding for the product, one for the difference
 *   firing_rates += s.float().squeeze()            one rounding
 *   _, idx = F.max_pool3d(firing_rates, ..., return_indices=True)
 *   out = s.flatten(2).gather(2, idx.flatten(2))   the spike at the window's first maximum
 * F.max_pool3d's CPU kernel scans the window's valid elements in (d, h, w) row-major order and keeps the first one unless
 * a later one compares strictly greater (or is a NaN).  Same arithmetic contract as the oracle (-ffp-contract=off).
 *
 *   gcc -O2 -fPIC -std=c11 -ffp-contract=off -fno-fast-math -fopenmp -shared -o libsnn_maxpool3d_oracle.so maxpool3d_oracle.c -lm
 */
#include "conv3d_oracle.c"

/* One axis of F.max_pool3d's geometry: the output size without ceil mode, padding at most half the kernel, and an
 * element of the input in every window. */
static int pool3_axis_ok(int in, int out, int k, int s, int p, int d) {
    if (in < 1 || k < 1 || s < 1 || d < 1 || p < 0 || p > k / 2) return 0;
    const int e = in + 2 * p - d * (k - 1) - 1;
    if (e < 0 || out != e / s + 1) return 0;
    for (int o = 0; o < out; ++o) {
        int any = 0;
        for (int j = 0; j < k; ++j) any |= o * s - p + j * d >= 0 && o * s - p + j * d < in;
        if (!any) return 0;
    }
    return 1;
}

/* include/snn_b200.h's conditions on a 3-D pooling connection. */
static int pool3_check(const snn_conn_t *C, int n_src, int n_tgt) {
    if (C->w || C->b || !C->pool_rates) return SNN_ERR_BAD_ARG;
    if (C->rule != SNN_RULE_NOOP || C->has_norm || C->mask) return SNN_ERR_UNSUPPORTED;
    if (C->cin != C->cout || C->cin < 1 || C->cin * C->din * C->hin * C->win != n_src || C->cout * C->dout * C->hout * C->wout != n_tgt)
        return SNN_ERR_BAD_ARG;
    if (!pool3_axis_ok(C->din, C->dout, C->kd, C->sd, C->pd, C->dd) || !pool3_axis_ok(C->hin, C->hout, C->kh, C->sh, C->ph, C->dh) ||
        !pool3_axis_ok(C->win, C->wout, C->kw, C->sw, C->pw, C->dw))
        return SNN_ERR_BAD_ARG;
    return SNN_OK;
}

/* One compute call: the rates of every sample advance by its spikes, then each target neuron takes the spike at its
 * window's first maximum; the result is added into `cur` like network.py:248. */
static void pool3_compute(const snn_conn_t *C, const uint8_t *s, int B, float *cur) {
    const int V = C->din * C->hin * C->win, ns = C->cin * V, L = C->dout * C->hout * C->wout, nt = C->cout * L;
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
            const int ch = j / L, l = j % L, oz = l / (C->hout * C->wout), oy = (l / C->wout) % C->hout, ox = l % C->wout;
            const float *rc = r + (size_t)ch * V;
            float best = 0.0f;
            int idx = -1;
            for (int kz = 0; kz < C->kd; ++kz) {
                const int iz = oz * C->sd - C->pd + kz * C->dd;
                if (iz < 0 || iz >= C->din) continue;
                for (int ky = 0; ky < C->kh; ++ky) {
                    const int iy = oy * C->sh - C->ph + ky * C->dh;
                    if (iy < 0 || iy >= C->hin) continue;
                    for (int kx = 0; kx < C->kw; ++kx) {
                        const int ix = ox * C->sw - C->pw + kx * C->dw;
                        if (ix < 0 || ix >= C->win) continue;
                        const int e = (iz * C->hin + iy) * C->win + ix;
                        const float v = rc[e];
                        if (idx < 0 || v > best || isnan(v)) { best = v; idx = e; }
                    }
                }
            }
            const float p = (idx >= 0 && sb[(size_t)ch * V + idx]) ? 1.0f : 0.0f;
            cur[(size_t)b * nt + j] = cur[(size_t)b * nt + j] + p;
        }
    }
}

static void any_mp3_compute(const snn_net_t *net, int c, const snn_run_opts_t *o, float *cur, int dense) {
    const snn_conn_t *C = &net->conns[c];
    if (C->kind == SNN_CONN_MAXPOOL3D) pool3_compute(C, net->layers[C->src].s, o->B, cur);
    else any_compute(net, c, o, cur, dense);
}

int snn_oracle_mp3_run_window(const snn_net_t *net, const snn_run_opts_t *o, int dense, int threads);
int snn_oracle_mp3_conn_compute(const snn_conn_t *C, int32_t n_src, int32_t n_tgt, int32_t B, const uint8_t *s, float *out);

/* Network.run (network.py:252-465): conv3d_oracle.c's timestep loop with the 3-D pooling connection in _get_inputs. */
int snn_oracle_mp3_run_window(const snn_net_t *net, const snn_run_opts_t *o, int dense, int threads) {
    if (!net || !o || net->n_conns < 0 || net->n_conns > SNN_MAX_CONNS || net->n_layers < 1 || net->n_layers > SNN_MAX_LAYERS) return SNN_ERR_BAD_ARG;
    int any = 0;
    for (int c = 0; c < net->n_conns; ++c) any |= net->conns[c].kind == SNN_CONN_MAXPOOL3D;
    if (!any) return snn_oracle_run_window(net, o, dense, threads);
    /* the oracle's own plan checks on everything but the Conv3d and 3-D pooling connections, which are checked here */
    snn_net_t rest = *net;
    rest.n_conns = 0;
    for (int c = 0; c < net->n_conns; ++c) {
        const snn_conn_t *C = &net->conns[c];
        if (C->kind != SNN_CONN_MAXPOOL3D && C->kind != SNN_CONN_CONV3D) { rest.conns[rest.n_conns++] = *C; continue; }
        if (C->src < 0 || C->src >= net->n_layers || C->tgt < 0 || C->tgt >= net->n_layers) return SNN_ERR_BAD_ARG;
        if (net->layers[C->tgt].kind == SNN_NODE_INPUT) return SNN_ERR_UNSUPPORTED;
        const int rc = C->kind == SNN_CONN_MAXPOOL3D ? pool3_check(C, net->layers[C->src].n, net->layers[C->tgt].n)
                                                     : conv3d_check(C, net->layers[C->src].n, net->layers[C->tgt].n, net->learning);
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
        if (SNN_RULE_IS_STDP(C->rule) && C->kind != SNN_CONN_CONV2D && C->kind != SNN_CONN_CONV3D) {
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
            any_mp3_compute(net, c, o, lws[C->tgt].cur, dense);
        }
        /* 2. layers in insertion order (network.py:386-429); one-step mode recomputes a layer's input just before it */
        for (int l = 0; l < net->n_layers; ++l) {
            if (o->one_step)
                for (int c = 0; c < net->n_conns; ++c) {
                    const snn_conn_t *C = &net->conns[c];
                    if (C->tgt != l) continue;
                    if (!lws[l].has_in) { memset(lws[l].cur, 0, sizeof(float) * (size_t)B * net->layers[l].n); lws[l].has_in = 1; }
                    any_mp3_compute(net, c, o, lws[l].cur, dense);
                }
            layer_forward(net, l, o, t, &lws[l], &err);
        }
        /* 3. connection updates in insertion order (network.py:431-454); a pooling connection has nothing to update */
        if (net->learning)
            for (int c = 0; c < net->n_conns; ++c) {
                const snn_conn_t *C = &net->conns[c];
                if (C->kind == SNN_CONN_MAXPOOL3D) continue;
                if (C->kind == SNN_CONN_CONV3D) conv3d_update(C);
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
    /* network.py:464-465; MaxPoo3dConnection.normalize does nothing (topology.py:1286-1291) */
    if (o->normalize)
        for (int c = 0; c < net->n_conns; ++c) {
            const snn_conn_t *C = &net->conns[c];
            if (C->kind == SNN_CONN_MAXPOOL3D || !C->has_norm) continue;
            if (C->kind == SNN_CONN_CONV3D) conv3d_normalize(C);
            else if (C->kind == SNN_CONN_CONV2D) normalize_conv(C);
            else normalize_cols(C->w, net->layers[C->src].n, net->layers[C->tgt].n, C->norm_abs, C->norm);
        }
    for (int l = 0; l < net->n_layers; ++l) { free(lws[l].cur); free(lws[l].cand); }
    for (int c = 0; c < net->n_conns; ++c) { free(cws[c].U); free(cws[c].V); free(cws[c].tx); free(cws[c].row_t); free(cws[c].col_t); }
    if (o->err_flag) *o->err_flag |= err;
    return SNN_OK;
}

/* MaxPoo3dConnection.compute: the rates in C->pool_rates advance in place, out is [B, C, dout, hout, wout]. */
int snn_oracle_mp3_conn_compute(const snn_conn_t *C, int32_t n_src, int32_t n_tgt, int32_t B, const uint8_t *s, float *out) {
    if (!C || C->kind != SNN_CONN_MAXPOOL3D) return snn_oracle_conn_compute(C, n_src, n_tgt, B, s, out);
    if (!s || !out || B <= 0) return SNN_ERR_BAD_ARG;
    const int rc = pool3_check(C, n_src, n_tgt);
    if (rc) return rc;
    memset(out, 0, sizeof(float) * (size_t)B * n_tgt);
    pool3_compute(C, s, B, out);
    return SNN_OK;
}
