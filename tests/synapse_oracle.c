/*
 * synapse_oracle.c — TEST INFRASTRUCTURE: the CPU oracle (oracle/snn_oracle.c, included unchanged) extended by a dense
 * Connection's per-synapse tensors (snn_conn_t wmin_t / wmax_t / nu0_t / nu1_t, include/snn_b200.h): wmin / wmax of any
 * shape that broadcasts to w (topology.py:74-81) and a learning rule's pair of rate tensors (learning.py:58-67).  It
 * exports the oracle's own entry points, so it is a drop-in superset of libsnn_oracle.so: plans without such tensors go
 * to the oracle's code untouched.
 *
 * Each update below is the oracle's own (conn_update, mstdp_dense_update, mstdpet_dense_update), op for op, with the
 * element (i, j) of a tensor where the oracle reads a scalar:
 *   clamp         w.clamp_(wmin, wmax) elementwise (learning.py:97-104)
 *   PostPre       x_tgt * nu0[j] before the batch sum, s_tgt * nu1[j] inside it (learning.py:403-417)
 *   WDep          fl(fl(nu0[i,j] * U) * (w - wmin[i,j])), fl(fl(nu1[i,j] * V) * (wmax[i,j] - w)) (learning.py:640-651)
 *   Hebbian       w + nu0[i,j] * U, w + nu1[i,j] * V (learning.py:1124-1134)
 *   MSTDP         w + nu0[i,j] * upd (learning.py:1562)
 *   MSTDPET       w + ((nu0[i,j] * dt) * reward) * e_trace (learning.py:2232-2238), dt = dt_scale
 * With rate tensors, the scalars nu0 / nu1 are the rule's gates (snn_b200.h).
 *
 *   gcc -O2 -fPIC -std=c11 -ffp-contract=off -fno-fast-math -fopenmp -shared -o libsnn_synapse_oracle.so synapse_oracle.c -lm
 */
#include "../include/snn_b200.h"

/* The oracle's window and single-operator update keep their code but not their symbols: these declarations give them
 * other assembler names, and the functions below take the exported ones. */
int snn_oracle_run_window(const snn_net_t *net, const snn_run_opts_t *o, int dense, int threads) __asm__("base_oracle_run_window");
int snn_oracle_conn_update(const snn_net_t *net, int32_t ci, int32_t B) __asm__("base_oracle_conn_update");
#include "../oracle/snn_oracle.c"

int syn_run_window(const snn_net_t *net, const snn_run_opts_t *o, int dense, int threads) __asm__("snn_oracle_run_window");
int syn_conn_update_entry(const snn_net_t *net, int32_t ci, int32_t B) __asm__("snn_oracle_conn_update");

static int has_syn(const snn_conn_t *C) { return C->kind == SNN_CONN_DENSE && (C->wmin_t || C->wmax_t || C->nu0_t || C->nu1_t); }

/* element (i, j) of a tensor in broadcast form `form`, or the scalar when there is none */
static inline float at(const float *t, int form, float scalar, int i, int j, int nt) {
    if (!t) return scalar;
    if (form == SNN_SYN_FULL) return t[(size_t)i * nt + j];
    if (form == SNN_SYN_TGT) return t[j];
    if (form == SNN_SYN_SRC) return t[i];
    return t[0];
}
#define WMIN(i, j) at(C->wmin_t, C->wmin_form, C->wmin, (i), (j), nt)
#define WMAX(i, j) at(C->wmax_t, C->wmax_form, C->wmax, (i), (j), nt)
#define NU0(i, j) at(C->nu0_t, C->nu0_form, C->nu0, (i), (j), nt)
#define NU1(i, j) at(C->nu1_t, C->nu1_form, C->nu1, (i), (j), nt)

static int syn_check(const snn_conn_t *C) {
    const float *t[4] = {C->wmin_t, C->wmax_t, C->nu0_t, C->nu1_t};
    const int f[4] = {C->wmin_form, C->wmax_form, C->nu0_form, C->nu1_form};
    for (int k = 0; k < 4; ++k)
        if (t[k] && (f[k] < SNN_SYN_FULL || f[k] > SNN_SYN_ONE)) return SNN_ERR_BAD_ARG;
    if ((C->nu0_t == NULL) != (C->nu1_t == NULL)) return SNN_ERR_BAD_ARG;
    if (C->rule == SNN_RULE_POSTPRE && C->nu0_t &&
        ((C->nu0_form != SNN_SYN_TGT && C->nu0_form != SNN_SYN_ONE) || (C->nu1_form != SNN_SYN_TGT && C->nu1_form != SNN_SYN_ONE)))
        return SNN_ERR_BAD_ARG;
    return SNN_OK;
}

/* conn_update (oracle/snn_oracle.c) of a dense connection with per-synapse tensors */
static void syn_conn_update(const snn_net_t *net, const snn_conn_t *C, const snn_run_opts_t *o, conn_ws_t *ws, int dense) {
    if (C->rule == SNN_RULE_NONE) return;
    const snn_layer_t *S = &net->layers[C->src], *G = &net->layers[C->tgt];
    const int B = o->B, ns = S->n, nt = G->n;
    float *w = C->w;
    const int stdp = SNN_RULE_IS_STDP(C->rule);
    const int hebb = C->rule == SNN_RULE_HEBBIAN;
    const int wdep = C->rule == SNN_RULE_WDEP_POSTPRE || hebb;
    const int pre_on = stdp && C->nu0 != 0.0f, post_on = stdp && C->nu1 != 0.0f;
    const float Bf = (float)B;
    int any_col = 0;

    if (pre_on) {
        float *tx = ws->tx;
        for (size_t k = 0; k < (size_t)B * nt; ++k) tx[k] = wdep ? G->x[k] : G->x[k] * NU0(0, (int)(k % nt));
#pragma omp parallel for schedule(static)
        for (int i = 0; i < ns; ++i) {
            float *Ui = ws->U + (size_t)i * nt;
            int touched = 0;
            if (dense) touched = 1;
            else for (int b = 0; b < B; ++b) if (S->s[(size_t)b * ns + i]) { touched = 1; break; }
            ws->row_t[i] = (uint8_t)touched;
            if (!touched) continue;
            for (int j = 0; j < nt; ++j) Ui[j] = 0.0f;
            for (int b = 0; b < B; ++b) {
                const uint8_t sb = S->s[(size_t)b * ns + i];
                if (!dense && !sb) continue;
                const float sv = sb ? 1.0f : 0.0f;
                const float *txb = tx + (size_t)b * nt;
                for (int j = 0; j < nt; ++j) Ui[j] = Ui[j] + sv * txb[j];
            }
            if (C->reduction == SNN_REDUCE_MEAN) for (int j = 0; j < nt; ++j) Ui[j] = Ui[j] / Bf;
        }
    } else memset(ws->row_t, 0, (size_t)ns);

    if (post_on) {
        for (int j = 0; j < nt; ++j) {
            int touched = dense;
            if (!touched) for (int b = 0; b < B; ++b) if (G->s[(size_t)b * nt + j]) { touched = 1; break; }
            ws->col_t[j] = (uint8_t)touched;
            any_col |= touched;
        }
        if (any_col) {
#pragma omp parallel for schedule(static)
            for (int i = 0; i < ns; ++i) {
                float *Vi = ws->V + (size_t)i * nt;
                for (int j = 0; j < nt; ++j) if (ws->col_t[j]) Vi[j] = 0.0f;
                for (int b = 0; b < B; ++b) {
                    const float xs = S->x[(size_t)b * ns + i];
                    const uint8_t *sg = G->s + (size_t)b * nt;
                    for (int j = 0; j < nt; ++j) {
                        if (!ws->col_t[j]) continue;
                        if (!dense && !sg[j]) continue;
                        const float ts = wdep ? (sg[j] ? 1.0f : 0.0f) : (sg[j] ? 1.0f : 0.0f) * NU1(0, j);
                        Vi[j] = Vi[j] + xs * ts;
                    }
                }
                if (C->reduction == SNN_REDUCE_MEAN) for (int j = 0; j < nt; ++j) if (ws->col_t[j]) Vi[j] = Vi[j] / Bf;
            }
        }
    } else memset(ws->col_t, 0, (size_t)nt);

    /* untouched entries stay as they are once every weight sits inside its own bounds (the full pass of the first
     * update of the window), as in the oracle */
    const int decay_on = C->weight_decay != 0.0f && C->weight_decay != 1.0f;
    const int full = dense || decay_on || (C->has_clamp && !ws->first_update_done);
    ws->first_update_done = 1;
#pragma omp parallel for schedule(static)
    for (int i = 0; i < ns; ++i) {
        const int rt = ws->row_t[i];
        if (!full && !rt && !any_col) continue;
        float *wi = w + (size_t)i * nt;
        const float *Ui = ws->U + (size_t)i * nt, *Vi = ws->V + (size_t)i * nt;
        for (int j = 0; j < nt; ++j) {
            const int ct = ws->col_t[j];
            if (!full && !rt && !ct) continue;
            float x = wi[j];
            if (hebb) {
                if (pre_on) x = x + NU0(i, j) * (rt ? Ui[j] : 0.0f);
                if (post_on) x = x + NU1(i, j) * (ct ? Vi[j] : 0.0f);
            } else if (wdep) {
                float upd = 0.0f;
                if (pre_on) upd = upd - (NU0(i, j) * (rt ? Ui[j] : 0.0f)) * (x - WMIN(i, j));
                if (post_on) upd = upd + (NU1(i, j) * (ct ? Vi[j] : 0.0f)) * (WMAX(i, j) - x);
                x = x + upd;
            } else {
                if (pre_on && rt) x = x - Ui[j];
                if (post_on && ct) x = x + Vi[j];
            }
            if (C->weight_decay != 0.0f) x = x * C->weight_decay;
            if (C->has_clamp) x = clampf(x, WMIN(i, j), WMAX(i, j));
            wi[j] = x;
        }
    }
}

/* mstdp_dense_update / mstdpet_dense_update (oracle/snn_oracle.c) with per-synapse tensors */
static void syn_mstdp_update(const snn_net_t *net, const snn_conn_t *C, const snn_run_opts_t *o, int dense) {
    const snn_layer_t *S = &net->layers[C->src], *G = &net->layers[C->tgt];
    const int ns = S->n, nt = G->n;
    const int et = C->rule == SNN_RULE_MSTDPET;
    const int B = et ? 1 : o->B;
    const float Bf = (float)B;
#pragma omp parallel for schedule(static)
    for (int i = 0; i < ns; ++i)
        for (int j = 0; j < nt; ++j) {
            const size_t k = (size_t)i * nt + j;
            float x;
            if (et) {
                const float e = C->p_plus[i] * (C->mst_spost[j] ? 1.0f : 0.0f) + (C->mst_spre[i] ? 1.0f : 0.0f) * C->p_minus[j];
                float tr = C->e_trace[k] * C->e_trace_decay;
                tr = tr + e / C->tc_e_trace;
                C->e_trace[k] = tr;
                const float coef = C->nu0_t ? (NU0(i, j) * C->dt_scale) * C->reward : C->et_coef;
                x = C->w[k] + coef * tr;
            } else {
                float upd = 0.0f;
                for (int b = 0; b < B; ++b) {
                    const uint8_t ss = C->mst_spre[(size_t)b * ns + i], sp = C->mst_spost[(size_t)b * nt + j];
                    if (!dense && !ss && !sp) continue;
                    const float e = C->p_plus[(size_t)b * ns + i] * (sp ? 1.0f : 0.0f) + (ss ? 1.0f : 0.0f) * C->p_minus[(size_t)b * nt + j];
                    upd = upd + C->reward * e;
                }
                if (C->reduction == SNN_REDUCE_MEAN) upd = upd / Bf;
                x = C->w[k] + NU0(i, j) * upd;
            }
            if (C->weight_decay != 0.0f) x = x * C->weight_decay;
            if (C->has_clamp) x = clampf(x, WMIN(i, j), WMAX(i, j));
            C->w[k] = x;
        }
    for (size_t k = 0; k < (size_t)B * ns; ++k) {
        const float x = C->p_plus[k] * C->p_plus_decay;
        C->p_plus[k] = x + C->a_plus * (S->s[k] ? 1.0f : 0.0f);
        C->mst_spre[k] = S->s[k] ? 1 : 0;
    }
    for (size_t k = 0; k < (size_t)B * nt; ++k) {
        const float x = C->p_minus[k] * C->p_minus_decay;
        C->p_minus[k] = x + C->a_minus * (G->s[k] ? 1.0f : 0.0f);
        C->mst_spost[k] = G->s[k] ? 1 : 0;
    }
}

/* Network.run (network.py:252-465): the oracle's timestep loop, with the updates above for the connections that carry
 * tensors. */
int syn_run_window(const snn_net_t *net, const snn_run_opts_t *o, int dense, int threads) {
    if (!net || !o) return SNN_ERR_BAD_ARG;
    int any = 0;
    for (int c = 0; c < net->n_conns && c < SNN_MAX_CONNS; ++c) {
        if (!has_syn(&net->conns[c])) continue;
        any = 1;
        const int rc = syn_check(&net->conns[c]);
        if (rc) return rc;
    }
    if (!any) return snn_oracle_run_window(net, o, dense, threads);
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
            layer_forward(net, l, o, t, &lws[l], &err);
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

/* connection.update(learning=True) from the layers' current s / x (topology.py:112-139) */
int syn_conn_update_entry(const snn_net_t *net, int32_t ci, int32_t B) {
    if (!net || ci < 0 || ci >= net->n_conns) return SNN_ERR_BAD_ARG;
    const snn_conn_t *C = &net->conns[ci];
    if (!has_syn(C)) return snn_oracle_conn_update(net, ci, B);
    const int rc = syn_check(C);
    if (rc) return rc;
    const int ns = net->layers[C->src].n, nt = net->layers[C->tgt].n;
    conn_ws_t ws; memset(&ws, 0, sizeof(ws));
    ws.U = (float *)calloc((size_t)ns * nt, sizeof(float));
    ws.V = (float *)calloc((size_t)ns * nt, sizeof(float));
    ws.tx = (float *)calloc((size_t)B * nt, sizeof(float));
    ws.row_t = (uint8_t *)calloc((size_t)ns, 1);
    ws.col_t = (uint8_t *)calloc((size_t)nt, 1);
    snn_run_opts_t o; memset(&o, 0, sizeof(o)); o.B = B; o.T = 1;
    syn_conn_update(net, C, &o, &ws, 0);
    free(ws.U); free(ws.V); free(ws.tx); free(ws.row_t); free(ws.col_t);
    return SNN_OK;
}
