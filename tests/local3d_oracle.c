/*
 * local3d_oracle.c — TEST INFRASTRUCTURE: the CPU oracle extended by LocalConnection2D (tests/local2d_oracle.c, which
 * includes oracle/snn_oracle.c; both included unchanged) and by LocalConnection3D (SNN_CONN_LOCAL3D).  It exports
 * local2d_oracle.c's entry points as they are, and its own under the names snn_oracle_l3d_*, which tests/local3d_oracle.py
 * puts in the place of the oracle's: plans without a 3-D local connection go to local2d_oracle.c's functions untouched,
 * and a plan with both local kinds runs here.
 *
 * LocalConnection3D (topology.py:1770-1917), the reference's axes H, W, D on the fields din / hin / win (include/snn_b200.h),
 * w [cin, n, K], n = n_filters * P, P = dout * hout * wout, K = kd * kh * kw:
 *   compute    target n' = f * P + p sees window p = (oz * hout + oy) * wout + ox: sum over ci ascending of (sum over k
 *              ascending of the spiking s[ci, oz*sd + kz, oy*sh + ky, ox*sw + kx] * w[ci, n', k], from +0),
 *              k = (kz * kh + ky) * kw + kx                                       (s_unfold * w).sum(-1).sum(1)
 *   rules      element (n', m), m < cin * K, is flat weight n' * cin * K + m; its source is the unfolded source at flat
 *              position (n' % P) * cin * K + m in [cin, P, K] order (the reference reshapes [cin, P, K] to [P, cin * K]
 *              and repeats it n_filters times, learning.py:322-388, 793-871, 1249-1314);
 *              pre = reduce_b x_tgt[b, n'] * s_src[b, src], post = reduce_b s_tgt[b, n'] * x_src[b, src], b ascending;
 *              then PostPre / WeightDependentPostPre / Hebbian as on a Conv2dConnection, decay and clamp (:87-104)
 *   normalize  each row of w viewed as [cin * n, K]: row *= (1 / row sum) * norm, sum ascending; no guard against a zero
 *              sum
 * Same arithmetic contract as the oracle (-ffp-contract=off).
 *
 *   gcc -O2 -fPIC -std=c11 -ffp-contract=off -fno-fast-math -fopenmp -shared -o libsnn_local3d_oracle.so local3d_oracle.c -lm
 */
#include "local2d_oracle.c"

/* include/snn_b200.h's conditions on a 3-D local connection. */
static int local3_check(const snn_conn_t *C, int n_src, int n_tgt) {
    if (!C->w || C->b) return SNN_ERR_BAD_ARG;
    if (C->cin < 1 || C->cout < 1 || C->kd < 1 || C->kh < 1 || C->kw < 1 || C->sd < 1 || C->sh < 1 || C->sw < 1) return SNN_ERR_BAD_ARG;
    if (C->pd || C->ph || C->pw || C->dh != 1 || C->dw != 1 || C->kd > C->din || C->kh > C->hin || C->kw > C->win) return SNN_ERR_BAD_ARG;
    if (C->dout != (C->din - C->kd) / C->sd + 1 || C->hout != (C->hin - C->kh) / C->sh + 1 || C->wout != (C->win - C->kw) / C->sw + 1)
        return SNN_ERR_BAD_ARG;
    if (C->cin * C->din * C->hin * C->win != n_src || C->cout * C->dout * C->hout * C->wout != n_tgt) return SNN_ERR_BAD_ARG;
    if (C->rule != SNN_RULE_NONE && C->rule != SNN_RULE_NOOP && C->rule != SNN_RULE_POSTPRE && C->rule != SNN_RULE_WDEP_POSTPRE &&
        C->rule != SNN_RULE_HEBBIAN)
        return SNN_ERR_UNSUPPORTED;
    if (C->mask) return SNN_ERR_UNSUPPORTED;
    return SNN_OK;
}

/* source neuron of window position l, kernel position k */
static int local3_at(const snn_conn_t *C, int ci, int l, int k) {
    const int HW = C->hout * C->wout, KHW = C->kh * C->kw;
    const int oz = l / HW, oy = (l % HW) / C->wout, ox = l % C->wout, kz = k / KHW, ky = (k % KHW) / C->kw, kx = k % C->kw;
    return ((ci * C->din + oz * C->sd + kz) * C->hin + oy * C->sh + ky) * C->win + ox * C->sw + kx;
}

static void local3_compute(const snn_conn_t *C, const uint8_t *s, int B, int ns, float *cur, int dense) {
    const int P = C->dout * C->hout * C->wout, nt = C->cout * P, K = C->kd * C->kh * C->kw;
#pragma omp parallel for schedule(static)
    for (int b = 0; b < B; ++b) {
        const uint8_t *sb = s + (size_t)b * ns;
        for (int j = 0; j < nt; ++j) {
            float p = 0.0f;
            for (int ci = 0; ci < C->cin; ++ci) {
                const float *wr = C->w + ((size_t)ci * nt + j) * K;
                float q = 0.0f;
                for (int k = 0; k < K; ++k) {
                    const uint8_t sv = sb[local3_at(C, ci, j % P, k)];
                    if (!dense && !sv) continue;
                    q = q + (sv ? 1.0f : 0.0f) * wr[k];
                }
                p = p + q;
            }
            cur[(size_t)b * nt + j] = cur[(size_t)b * nt + j] + p;
        }
    }
}

static int local3_source(const snn_conn_t *C, int n, int m) {
    const int K = C->kd * C->kh * C->kw, P = C->dout * C->hout * C->wout;
    const int q = (n % P) * C->cin * K + m, ci = q / (P * K), r = q % (P * K);
    return local3_at(C, ci, r / K, r % K);
}

static void local3_update(const snn_layer_t *S, const snn_layer_t *G, const snn_conn_t *C, int B) {
    const int nt = G->n, ns = S->n, M = C->cin * C->kd * C->kh * C->kw;
    const size_t NW = (size_t)nt * M;
    if (!SNN_RULE_IS_STDP(C->rule)) {   /* learning.NoOp: decay only (learning.py:93-94) */
        if (C->rule == SNN_RULE_NOOP && C->weight_decay != 0.0f)
            for (size_t e = 0; e < NW; ++e) C->w[e] = C->w[e] * C->weight_decay;
        return;
    }
    const int hebb = C->rule == SNN_RULE_HEBBIAN;
    const int pre_on = C->nu0 != 0.0f || hebb, post_on = C->nu1 != 0.0f || hebb;
#pragma omp parallel for schedule(static)
    for (int n = 0; n < nt; ++n)
        for (int m = 0; m < M; ++m) {
            const int src = local3_source(C, n, m);
            float U = 0.0f, V = 0.0f;
            for (int b = 0; b < B; ++b) {
                if (pre_on && S->s[(size_t)b * ns + src]) U = U + G->x[(size_t)b * nt + n];
                if (post_on && G->s[(size_t)b * nt + n]) V = V + S->x[(size_t)b * ns + src];
            }
            if (C->reduction == SNN_REDUCE_MEAN) { U = U / (float)B; V = V / (float)B; }
            const size_t e = (size_t)n * M + m;
            float x = C->w[e];
            if (C->rule == SNN_RULE_WDEP_POSTPRE) {
                float upd = 0.0f;
                if (pre_on) upd = upd - (C->nu0 * U) * (x - C->wmin);      /* learning.py:853-859 */
                if (post_on) upd = upd + (C->nu1 * V) * (C->wmax - x);     /* :861-869 */
                x = x + upd;
            } else if (hebb) {
                x = x + C->nu0 * U;                                        /* learning.py:1308 */
                x = x + C->nu1 * V;                                        /* :1312 */
            } else {
                if (pre_on) x = x - C->nu0 * U;                            /* learning.py:380-382 */
                if (post_on) x = x + C->nu1 * V;                           /* :384-386 */
            }
            if (C->weight_decay != 0.0f) x = x * C->weight_decay;
            if (C->has_clamp) x = clampf(x, C->wmin, C->wmax);
            C->w[e] = x;
        }
}

static void local3_normalize(const snn_conn_t *C, int n_tgt) {
    const int K = C->kd * C->kh * C->kw, rows = C->cin * n_tgt;
    for (int r = 0; r < rows; ++r) {
        float *w = C->w + (size_t)r * K;
        float tot = 0.0f;
        for (int k = 0; k < K; ++k) tot = tot + w[k];
        const float fac = (1.0f / tot) * C->norm;
        for (int k = 0; k < K; ++k) w[k] = w[k] * fac;
    }
}

static void any3_compute(const snn_net_t *net, int c, const snn_run_opts_t *o, float *cur, int dense) {
    const snn_conn_t *C = &net->conns[c];
    const snn_layer_t *S = &net->layers[C->src];
    if (C->kind == SNN_CONN_LOCAL3D) local3_compute(C, S->s, o->B, S->n, cur, dense);
    else any_compute(net, c, o, cur, dense);
}

static int is_local(const snn_conn_t *C) { return C->kind == SNN_CONN_LOCAL2D || C->kind == SNN_CONN_LOCAL3D; }

int snn_oracle_l3d_run_window(const snn_net_t *net, const snn_run_opts_t *o, int dense, int threads);
int snn_oracle_l3d_conn_compute(const snn_conn_t *C, int32_t n_src, int32_t n_tgt, int32_t B, const uint8_t *s, float *out);
int snn_oracle_l3d_conn_update(const snn_net_t *net, int32_t ci, int32_t B);
int snn_oracle_l3d_conn_normalize(const snn_conn_t *C, int32_t n_src, int32_t n_tgt);

/* Network.run (network.py:252-465): local2d_oracle.c's timestep loop with either local connection in _get_inputs, the
 * update and the end-of-run normalize. */
int snn_oracle_l3d_run_window(const snn_net_t *net, const snn_run_opts_t *o, int dense, int threads) {
    if (!net || !o || net->n_conns < 0 || net->n_conns > SNN_MAX_CONNS || net->n_layers < 1 || net->n_layers > SNN_MAX_LAYERS) return SNN_ERR_BAD_ARG;
    int any = 0;
    for (int c = 0; c < net->n_conns; ++c) any |= net->conns[c].kind == SNN_CONN_LOCAL3D;
    if (!any) return snn_oracle_run_window(net, o, dense, threads);
    /* the oracle's own plan checks on everything but the local connections, which are checked here */
    snn_net_t rest = *net;
    rest.n_conns = 0;
    for (int c = 0; c < net->n_conns; ++c) {
        const snn_conn_t *C = &net->conns[c];
        if (!is_local(C)) { rest.conns[rest.n_conns++] = *C; continue; }
        if (C->src < 0 || C->src >= net->n_layers || C->tgt < 0 || C->tgt >= net->n_layers) return SNN_ERR_BAD_ARG;
        if (net->layers[C->tgt].kind == SNN_NODE_INPUT) return SNN_ERR_UNSUPPORTED;
        const int rc = C->kind == SNN_CONN_LOCAL3D ? local3_check(C, net->layers[C->src].n, net->layers[C->tgt].n)
                                                   : local_check(C, net->layers[C->src].n, net->layers[C->tgt].n);
        if (rc) return rc;
        if (SNN_RULE_IS_STDP(C->rule) && (!net->layers[C->src].traces || !net->layers[C->tgt].traces)) return SNN_ERR_BAD_ARG;
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
        if (SNN_RULE_IS_STDP(C->rule) && C->kind != SNN_CONN_CONV2D && !is_local(C)) {
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
            any3_compute(net, c, o, lws[C->tgt].cur, dense);
        }
        /* 2. layers in insertion order (network.py:386-429); one-step mode recomputes a layer's input just before it */
        for (int l = 0; l < net->n_layers; ++l) {
            if (o->one_step)
                for (int c = 0; c < net->n_conns; ++c) {
                    const snn_conn_t *C = &net->conns[c];
                    if (C->tgt != l) continue;
                    if (!lws[l].has_in) { memset(lws[l].cur, 0, sizeof(float) * (size_t)B * net->layers[l].n); lws[l].has_in = 1; }
                    any3_compute(net, c, o, lws[l].cur, dense);
                }
            layer_forward(net, l, o, t, &lws[l], &err);
        }
        /* 3. connection updates in insertion order (network.py:431-454) */
        if (net->learning)
            for (int c = 0; c < net->n_conns; ++c) {
                const snn_conn_t *C = &net->conns[c];
                if (C->kind == SNN_CONN_LOCAL3D) local3_update(&net->layers[C->src], &net->layers[C->tgt], C, B);
                else if (C->kind == SNN_CONN_LOCAL2D) local_update(&net->layers[C->src], &net->layers[C->tgt], C, B);
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
    if (o->normalize)   /* network.py:464-465 */
        for (int c = 0; c < net->n_conns; ++c) {
            const snn_conn_t *C = &net->conns[c];
            if (!C->has_norm) continue;
            if (C->kind == SNN_CONN_LOCAL3D) local3_normalize(C, net->layers[C->tgt].n);
            else if (C->kind == SNN_CONN_LOCAL2D) local_normalize(C, net->layers[C->tgt].n);
            else if (C->kind == SNN_CONN_CONV2D) normalize_conv(C);
            else normalize_cols(C->w, net->layers[C->src].n, net->layers[C->tgt].n, C->norm_abs, C->norm);
        }
    for (int l = 0; l < net->n_layers; ++l) { free(lws[l].cur); free(lws[l].cand); }
    for (int c = 0; c < net->n_conns; ++c) { free(cws[c].U); free(cws[c].V); free(cws[c].tx); free(cws[c].row_t); free(cws[c].col_t); }
    if (o->err_flag) *o->err_flag |= err;
    return SNN_OK;
}

int snn_oracle_l3d_conn_compute(const snn_conn_t *C, int32_t n_src, int32_t n_tgt, int32_t B, const uint8_t *s, float *out) {
    if (!C || C->kind != SNN_CONN_LOCAL3D) return snn_oracle_conn_compute(C, n_src, n_tgt, B, s, out);
    if (!s || !out || B <= 0) return SNN_ERR_BAD_ARG;
    const int rc = local3_check(C, n_src, n_tgt);
    if (rc) return rc;
    memset(out, 0, sizeof(float) * (size_t)B * n_tgt);
    local3_compute(C, s, B, n_src, out, 0);
    return SNN_OK;
}

int snn_oracle_l3d_conn_update(const snn_net_t *net, int32_t ci, int32_t B) {
    if (!net || ci < 0 || ci >= net->n_conns || net->conns[ci].kind != SNN_CONN_LOCAL3D) return snn_oracle_conn_update(net, ci, B);
    const snn_conn_t *C = &net->conns[ci];
    const int rc = local3_check(C, net->layers[C->src].n, net->layers[C->tgt].n);
    if (rc) return rc;
    local3_update(&net->layers[C->src], &net->layers[C->tgt], C, B);
    return SNN_OK;
}

int snn_oracle_l3d_conn_normalize(const snn_conn_t *C, int32_t n_src, int32_t n_tgt) {
    if (!C || C->kind != SNN_CONN_LOCAL3D) return snn_oracle_conn_normalize(C, n_src, n_tgt);
    if (!C->w) return SNN_ERR_BAD_ARG;
    if (C->has_norm) local3_normalize(C, n_tgt);
    return SNN_OK;
}
