/*
 * conv1d_oracle.c — TEST INFRASTRUCTURE: the CPU oracle (oracle/snn_oracle.c, included unchanged) extended by
 * Conv1dConnection (SNN_CONN_CONV1D).  It exports the oracle's own entry points, so it is a drop-in superset of
 * libsnn_oracle.so: plans without a Conv1dConnection go to the oracle's functions untouched.
 *
 * Conv1dConnection (topology.py:540-683), w [cout, cin, kw], b [cout], source [cin, win], target [cout, wout]:
 *   compute    target (co, ox): the sum of the taps whose zero-padded input position spiked, in ascending (ci, kx)
 *              order from +0, then + b[co]                                    F.conv1d(s.float(), w, b, stride, padding)
 *   rules      element (co, m), m < cin * kw, is flat weight co * cin * kw + m.  It pairs target position l' with the
 *              source neuron the reference's reshape of the unfolded source [cin, L, kw] to [L, cin * kw] puts at
 *              column m of row l' (learning.py:434-442): f = l' * cin * kw + m, c = f / (L * kw), l = (f % (L * kw)) / kw,
 *              kk = f % kw, source c * win + l * sw - pw + kk (a padding position: no term).
 *              pre = reduce_b sum_l' x_tgt[b, co, l'] * s_src[b, src], post = reduce_b sum_l' s_tgt[b, co, l'] * x_src[b, src]:
 *              each sample's sum over l' ascending from +0, the terms of silent spikes skipped, then the samples' sums in
 *              ascending b; then PostPre / WeightDependentPostPre / Hebbian as on a Conv2dConnection, decay and clamp
 *              (learning.py:422-455, 873-918, 1316-1346, :87-104)
 *   normalize  each row of w viewed as [cout * cin, kw]: row *= norm / (row sum, ascending), like the oracle's
 *              Conv2dConnection normalize; no guard against a zero sum
 * Same arithmetic contract as the oracle (-ffp-contract=off).
 *
 *   gcc -O2 -fPIC -std=c11 -ffp-contract=off -fno-fast-math -fopenmp -shared -o libsnn_conv1d_oracle.so conv1d_oracle.c -lm
 */
#define snn_oracle_run_window oracle_run_window_base
#define snn_oracle_conn_compute oracle_conn_compute_base
#define snn_oracle_conn_update oracle_conn_update_base
#define snn_oracle_conn_normalize oracle_conn_normalize_base
#include "../oracle/snn_oracle.c"
#undef snn_oracle_run_window
#undef snn_oracle_conn_compute
#undef snn_oracle_conn_update
#undef snn_oracle_conn_normalize

int snn_oracle_run_window(const snn_net_t *net, const snn_run_opts_t *o, int dense, int threads);
int snn_oracle_conn_compute(const snn_conn_t *C, int32_t n_src, int32_t n_tgt, int32_t B, const uint8_t *s, float *out);
int snn_oracle_conn_update(const snn_net_t *net, int32_t ci, int32_t B);
int snn_oracle_conn_normalize(const snn_conn_t *C, int32_t n_src, int32_t n_tgt);

/* include/snn_b200.h's conditions on a Conv1dConnection. */
static int conv1d_check(const snn_conn_t *C, int n_src, int n_tgt) {
    if (!C->w || !C->b) return SNN_ERR_BAD_ARG;
    if (C->cin < 1 || C->cout < 1 || C->kw < 1 || C->sw < 1 || C->pw < 0 || C->win < 1 || C->wout < 1) return SNN_ERR_BAD_ARG;
    if (C->hin != 1 || C->hout != 1 || C->kh != 1 || C->sh != 1 || C->ph != 0 || C->dh != 1 || C->dw != 1) return SNN_ERR_BAD_ARG;
    if (C->win + 2 * C->pw < C->kw || C->wout != (C->win - C->kw + 2 * C->pw) / C->sw + 1) return SNN_ERR_BAD_ARG;
    if ((long long)C->cin * C->win != n_src || (long long)C->cout * C->wout != n_tgt) return SNN_ERR_BAD_ARG;
    if (C->rule != SNN_RULE_NONE && C->rule != SNN_RULE_NOOP && C->rule != SNN_RULE_POSTPRE && C->rule != SNN_RULE_WDEP_POSTPRE &&
        C->rule != SNN_RULE_HEBBIAN)
        return SNN_ERR_UNSUPPORTED;
    if (C->mask) return SNN_ERR_UNSUPPORTED;
    return SNN_OK;
}

static void conv1d_compute(const snn_conn_t *C, const uint8_t *s, int B, int ns, float *cur, int dense) {
    const int nt = C->cout * C->wout;
#pragma omp parallel for schedule(static)
    for (int b = 0; b < B; ++b) {
        const uint8_t *sb = s + (size_t)b * ns;
        for (int j = 0; j < nt; ++j) {
            const int co = j / C->wout, ox = j % C->wout;
            const float *wf = C->w + (size_t)co * C->cin * C->kw;
            float p = 0.0f;
            for (int ci = 0; ci < C->cin; ++ci)
                for (int kx = 0; kx < C->kw; ++kx) {
                    const int ix = ox * C->sw - C->pw + kx;
                    if (ix < 0 || ix >= C->win) continue;
                    const uint8_t sv = sb[(size_t)ci * C->win + ix];
                    if (!dense && !sv) continue;
                    p = p + (sv ? 1.0f : 0.0f) * wf[ci * C->kw + kx];
                }
            cur[(size_t)b * nt + j] = cur[(size_t)b * nt + j] + (p + C->b[co]);
        }
    }
}

/* the source neuron paired with target position lt by element m, or -1 (a padding position) */
static int conv1d_source(const snn_conn_t *C, int lt, int m) {
    const int L = C->wout, K = C->kw;
    const long long f = (long long)lt * C->cin * K + m;
    const int c = (int)(f / ((long long)L * K)), r = (int)(f % ((long long)L * K)), l = r / K, kk = r % K;
    const int pos = l * C->sw - C->pw + kk;
    return pos < 0 || pos >= C->win ? -1 : c * C->win + pos;
}

static void conv1d_update(const snn_layer_t *S, const snn_layer_t *G, const snn_conn_t *C, int B) {
    const int ns = S->n, nt = G->n, M = C->cin * C->kw, L = C->wout;
    const int NW = C->cout * M;
    if (!SNN_RULE_IS_STDP(C->rule)) {   /* learning.NoOp: decay only (learning.py:93-94) */
        if (C->rule == SNN_RULE_NOOP && C->weight_decay != 0.0f)
            for (int e = 0; e < NW; ++e) C->w[e] = C->w[e] * C->weight_decay;
        return;
    }
    const int hebb = C->rule == SNN_RULE_HEBBIAN;
    const int pre_on = C->nu0 != 0.0f || hebb, post_on = C->nu1 != 0.0f || hebb;
#pragma omp parallel for schedule(static)
    for (int e = 0; e < NW; ++e) {
        const int co = e / M, m = e % M;
        float U = 0.0f, V = 0.0f;
        for (int b = 0; b < B; ++b) {
            float u1 = 0.0f, v1 = 0.0f;
            for (int lt = 0; lt < L; ++lt) {
                const int src = conv1d_source(C, lt, m);
                if (src < 0) continue;
                const size_t tj = (size_t)b * nt + (size_t)co * L + lt, si = (size_t)b * ns + src;
                if (pre_on && S->s[si]) u1 = u1 + G->x[tj];
                if (post_on && G->s[tj]) v1 = v1 + S->x[si];
            }
            U = U + u1;
            V = V + v1;
        }
        if (C->reduction == SNN_REDUCE_MEAN) { U = U / (float)B; V = V / (float)B; }
        float x = C->w[e];
        if (C->rule == SNN_RULE_WDEP_POSTPRE) {
            float upd = 0.0f;
            if (pre_on) upd = upd - (C->nu0 * U) * (x - C->wmin);      /* learning.py:899-905 */
            if (post_on) upd = upd + (C->nu1 * V) * (C->wmax - x);     /* :908-914 */
            x = x + upd;
        } else if (hebb) {
            x = x + C->nu0 * U;                                        /* learning.py:1339-1340 */
            x = x + C->nu1 * V;                                        /* :1343-1344 */
        } else {
            if (pre_on) x = x - C->nu0 * U;                            /* learning.py:446-448 */
            if (post_on) x = x + C->nu1 * V;                           /* :451-453 */
        }
        if (C->weight_decay != 0.0f) x = x * C->weight_decay;
        if (C->has_clamp) x = clampf(x, C->wmin, C->wmax);
        C->w[e] = x;
    }
}

static void conv1d_normalize(const snn_conn_t *C) {
    const int F = C->cout * C->cin, K = C->kw;
    for (int f = 0; f < F; ++f) {
        float *w = C->w + (size_t)f * K;
        float tot = 0.0f;
        for (int k = 0; k < K; ++k) tot = tot + w[k];
        const float fac = C->norm / tot;
        for (int k = 0; k < K; ++k) w[k] = w[k] * fac;
    }
}

static void any_compute(const snn_net_t *net, int c, const snn_run_opts_t *o, float *cur, int dense) {
    const snn_conn_t *C = &net->conns[c];
    const snn_layer_t *S = &net->layers[C->src];
    if (C->kind == SNN_CONN_CONV1D) conv1d_compute(C, S->s, o->B, S->n, cur, dense);
    else if (C->kind == SNN_CONN_CONV2D) conv_compute(C, S, o->B, cur, dense);
    else conn_compute(C, S, net->layers[C->tgt].n, o->B, cur, dense);
}

/* Network.run (network.py:252-465): oracle/snn_oracle.c's timestep loop with the Conv1dConnection in _get_inputs, the
 * update and the end-of-run normalize. */
int snn_oracle_run_window(const snn_net_t *net, const snn_run_opts_t *o, int dense, int threads) {
    if (!net || !o || net->n_conns < 0 || net->n_conns > SNN_MAX_CONNS || net->n_layers < 1 || net->n_layers > SNN_MAX_LAYERS) return SNN_ERR_BAD_ARG;
    int any = 0;
    for (int c = 0; c < net->n_conns; ++c) any |= net->conns[c].kind == SNN_CONN_CONV1D;
    if (!any) return oracle_run_window_base(net, o, dense, threads);
    /* the oracle's own plan checks on everything but the Conv1dConnections, which are checked here */
    snn_net_t rest = *net;
    rest.n_conns = 0;
    for (int c = 0; c < net->n_conns; ++c) {
        const snn_conn_t *C = &net->conns[c];
        if (C->kind != SNN_CONN_CONV1D) { rest.conns[rest.n_conns++] = *C; continue; }
        if (C->src < 0 || C->src >= net->n_layers || C->tgt < 0 || C->tgt >= net->n_layers) return SNN_ERR_BAD_ARG;
        if (net->layers[C->tgt].kind == SNN_NODE_INPUT) return SNN_ERR_UNSUPPORTED;
        const int rc = conv1d_check(C, net->layers[C->src].n, net->layers[C->tgt].n);
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
        if (SNN_RULE_IS_STDP(C->rule) && C->kind != SNN_CONN_CONV2D && C->kind != SNN_CONN_CONV1D) {
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
        /* 3. connection updates in insertion order (network.py:431-454) */
        if (net->learning)
            for (int c = 0; c < net->n_conns; ++c) {
                const snn_conn_t *C = &net->conns[c];
                if (C->kind == SNN_CONN_CONV1D) conv1d_update(&net->layers[C->src], &net->layers[C->tgt], C, B);
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
            if (C->kind == SNN_CONN_CONV1D) conv1d_normalize(C);
            else if (C->kind == SNN_CONN_CONV2D) normalize_conv(C);
            else normalize_cols(C->w, net->layers[C->src].n, net->layers[C->tgt].n, C->norm_abs, C->norm);
        }
    for (int l = 0; l < net->n_layers; ++l) { free(lws[l].cur); free(lws[l].cand); }
    for (int c = 0; c < net->n_conns; ++c) { free(cws[c].U); free(cws[c].V); free(cws[c].tx); free(cws[c].row_t); free(cws[c].col_t); }
    if (o->err_flag) *o->err_flag |= err;
    return SNN_OK;
}

int snn_oracle_conn_compute(const snn_conn_t *C, int32_t n_src, int32_t n_tgt, int32_t B, const uint8_t *s, float *out) {
    if (!C || C->kind != SNN_CONN_CONV1D) return oracle_conn_compute_base(C, n_src, n_tgt, B, s, out);
    if (!s || !out || B <= 0) return SNN_ERR_BAD_ARG;
    const int rc = conv1d_check(C, n_src, n_tgt);
    if (rc) return rc;
    memset(out, 0, sizeof(float) * (size_t)B * n_tgt);
    conv1d_compute(C, s, B, n_src, out, 0);
    return SNN_OK;
}

int snn_oracle_conn_update(const snn_net_t *net, int32_t ci, int32_t B) {
    if (!net || ci < 0 || ci >= net->n_conns || net->conns[ci].kind != SNN_CONN_CONV1D) return oracle_conn_update_base(net, ci, B);
    const snn_conn_t *C = &net->conns[ci];
    const int rc = conv1d_check(C, net->layers[C->src].n, net->layers[C->tgt].n);
    if (rc) return rc;
    conv1d_update(&net->layers[C->src], &net->layers[C->tgt], C, B);
    return SNN_OK;
}

int snn_oracle_conn_normalize(const snn_conn_t *C, int32_t n_src, int32_t n_tgt) {
    if (!C || C->kind != SNN_CONN_CONV1D) return oracle_conn_normalize_base(C, n_src, n_tgt);
    if (!C->w) return SNN_ERR_BAD_ARG;
    if (C->has_norm) conv1d_normalize(C);
    return SNN_OK;
}
