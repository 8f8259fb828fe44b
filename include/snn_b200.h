/*
 * snn_b200.h — C ABI of the CUDA-native SNN simulation core (H100, sm_90a).
 *
 * This is the drop-in boundary for ONE path of BindsNET: the per-timestep loop of
 * `Network.run()` (reference: bindsnet/network/network.py:252-465).  The reference has no
 * native code and therefore no FFI of its own; the entry points below are what a
 * maintainer would bind from `bindsnet/network/network.py` (see INTEGRATION.md for the
 * ctypes stub).  Everything is plain C: pointers, sizes, POD structs, no torch types.
 *
 * A *window* is one call of Network.run(inputs, time=T): T timesteps over a batch of B
 * samples.  The caller describes the network as an array of layers (reference: Nodes
 * subclasses, bindsnet/network/nodes.py) and an array of connections (reference:
 * AbstractConnection subclasses, bindsnet/network/topology.py) with their learning rule
 * (bindsnet/learning/learning.py, bindsnet/learning/MCC_learning.py), in the insertion
 * order of Network.add_layer / Network.add_connection, which fixes the accumulation order
 * (network.py:225,246-248,386).
 *
 * All state pointers are the storage of the user's own tensors (layer.v, layer.x,
 * connection.w ...) and are updated IN PLACE: after the call they hold the state the
 * reference would hold after run() (network.py:380-465), including the end-of-run
 * normalize (network.py:464-465).
 *
 * The same structs are consumed by two libraries:
 *   - libsnn_b200.so   (bindsnet_b200/csrc, CUDA sm_90a; every pointer is a DEVICE pointer)
 *   - libsnn_oracle.so (oracle/, plain C test infrastructure; every pointer is a HOST pointer)
 * (and by tests/emu/libsnn_emu.so, test infrastructure: the generic kernel's CUDA sources compiled for the host on a small
 * emulation of the CUDA execution model, HOST pointers).
 */
#ifndef SNN_B200_H
#define SNN_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SNN_ABI_VERSION 13
#define SNN_MAX_LAYERS 8
#define SNN_MAX_CONNS 12

/* ---- node kinds (reference: bindsnet/network/nodes.py) ---- */
#define SNN_NODE_INPUT 0 /* Input            nodes.py:172-228  */
#define SNN_NODE_LIF 1   /* LIFNodes         nodes.py:418-559  */
#define SNN_NODE_DC 2    /* DiehlAndCookNodes nodes.py:981-1144; with one_spike = 0 also AdaptiveLIFNodes nodes.py:829-978
                            (the same arithmetic: decay, theta decay, gated input, threshold + theta, theta += plus * sum_b s) */
#define SNN_NODE_IF 3         /* IFNodes          nodes.py:308-415: no leak, gate taken before the refractory decrement */
#define SNN_NODE_CURRENT_LIF 4 /* CurrentLIFNodes nodes.py:681-826: decaying synaptic current i, gate taken after the decrement */
#define SNN_NODE_BOOSTED_LIF 5 /* BoostedLIFNodes nodes.py:562-678: LIF without rest / reset / lbound: v *= decay, reset to 0 */
#define SNN_NODE_MCP 6         /* McCullochPitts  nodes.py:231-305: v = x, s = v >= thresh; no refractory state (refrac_count NULL) */
#define SNN_NODE_SUBIF 7       /* conversion.SubtractiveResetIFNodes conversion/nodes.py:73-99, one rounding per op:
                                    v  = v + (rc == 0) * x          (-0.0 == 0 counts as 0)
                                    rc = (rc > 0) * (rc - dt)       (rc <= 0 gives -0.0; 0 < rc < dt a negative rc, which
                                                                     gates the NEXT step's input off)
                                    s  = v >= thresh;  s ? rc = refrac, v = v - thresh   (reset by subtraction)
                                    v  = max(v, lbound) if has_lbound;  then traces and summed += x as for every kind.
                                  Generic tier only */
#define SNN_NODE_PASSTHROUGH 8 /* conversion.PassThroughNodes conversion/nodes.py:137-144: s = x, nothing else (no trace or
                                  summed update whatever the flags say; v and refrac_count are NULL).  `s` points to
                                  FLOAT32 [B,n] holding 0.0 / 1.0 (the reference's s is the float input itself); a step whose
                                  x is not in {0, 1} raises SNN_ERR_NONBINARY.  The only connection into such a layer is an
                                  SNN_CONN_MAXPOOL2D, and a connection with such an endpoint has rule SNN_RULE_NONE or
                                  SNN_RULE_NOOP.  Generic tier only */
/* Per-neuron parameters of an SNN_NODE_LIF or SNN_NODE_DC layer (a parameter given to LIFNodes, AdaptiveLIFNodes or
 * DiehlAndCookNodes as a tensor, which the reference broadcasts elementwise against [B, *shape]).  The flag is OR-ed into
 * snn_layer_t.kind; such a layer's pn points to a float32 [k, n] block whose row r holds parameter r of every neuron
 * (r < k for every bit r of pn_mask) and takes the place of the scalar field wherever the layer reads it:
 *   SNN_PN_THRESH       thresh       s = v >= thresh[j]  (DC: v >= fl(thresh[j] + theta[j]))
 *   SNN_PN_REST         rest         v = fl(decay[j] * fl(v - rest[j])) + rest[j]
 *   SNN_PN_DECAY        decay        exp(-dt / tc_decay[j]) evaluated in fp32 like nodes.py:546-548
 *   SNN_PN_THETA_PLUS   theta_plus   theta[j] += fl(theta_plus[j] * count), count = the step's spikes summed over the batch (DC)
 *   SNN_PN_THETA_DECAY  theta_decay  theta[j] *= theta_decay[j] (DC)
 *   SNN_PN_TRACE_DECAY  trace_decay  x *= trace_decay[j]  (traces only)
 *   SNN_PN_TRACE_SCALE  trace_scale  x += fl(trace_scale[j] * s)  (traces_additive only: the reference's masked_fill_
 *                                    takes no tensor value)
 * A bit the kind does not have (THETA_* on SNN_NODE_LIF, TRACE_* without traces, TRACE_SCALE without traces_additive), a
 * NULL pn with a non-zero mask or a flag on another kind is SNN_ERR_BAD_ARG.  Generic tier only: tier 0 selects tier 1,
 * a forced tier 2 or 3 (and so a delta window) is SNN_ERR_UNSUPPORTED; not in a plan that also holds an SNN_CONN_SPARSE
 * connection, MCC features or a kind of the pooling instantiation.  A library older than the flag refuses such a plan
 * (it rejects every kind above SNN_NODE_PASSTHROUGH with SNN_ERR_UNSUPPORTED). */
#define SNN_NODE_PN 0x100
#define SNN_PN_THRESH 0
#define SNN_PN_REST 1
#define SNN_PN_DECAY 2
#define SNN_PN_THETA_PLUS 3
#define SNN_PN_THETA_DECAY 4
#define SNN_PN_TRACE_DECAY 5
#define SNN_PN_TRACE_SCALE 6
#define SNN_PN_ROWS 7

/* ---- connection kinds (reference: bindsnet/network/topology.py) ---- */
#define SNN_CONN_DENSE 0 /* Connection: s.float() @ w + b                topology.py:332-346 */
#define SNN_CONN_MCC 1   /* MulticompartmentConnection[Weight]: sum_i W*s  topology.py:437-479,
                            topology_features.py:633-645 (same maths, dt-scaled STDP)          */
#define SNN_CONN_CONV2D 2 /* Conv2dConnection: F.conv2d(s.float(), w, b, stride, padding, dilation)
                             topology.py:799-815; w is [Cout, Cin, kh, kw], b is [Cout]; the source layer's
                             neurons are indexed (ci, y, x), the target's (co, oy, ox), row-major */
#define SNN_CONN_SPARSE 3 /* SparseConnection: a Connection whose w is a torch.sparse_coo tensor, s.float() @ w + b
                             topology.py:2009-2017, :332-346.  w holds the nnz stored values in CSR order (sp_rowptr /
                             sp_col); out[b,j] = sum over the spiking i with a stored (i,j), i ascending, from +0, then
                             + b[j] — bit-identical to the dense gather over the same values.  Fixed pattern: rules
                             SNN_RULE_NONE / SNN_RULE_NOOP only (decay of the stored values), no normalize, no mask,
                             generic tier only */
#define SNN_CONN_MAXPOOL2D 4 /* MaxPool2dConnection: online-rate max pooling, topology.py:1124-1211.  No weights (w, b NULL),
                                rule SNN_RULE_NOOP only, no normalize, no mask.  Source [C,hin,win], target [C,hout,wout]
                                (the conv geometry fields with cin = cout = C; kh/kw, sh/sw, ph/pw, dh/dw as for
                                F.max_pool2d, no ceil mode).  Each compute:
                                  1. r = fl(r - fl(pool_decay * r)); r = fl(r + s)   on pool_rates [B,C,hin,win], in place
                                  2. idx = the first maximum of r[b,c] over the window, row-major window order, padding
                                     never chosen (strict >, so -0 == +0 ties keep the earlier element)
                                  3. out[b,c,oy,ox] = s[b,c,idx] as 0.0 / 1.0
                                Inside a window the rates read by step t fold in the spikes that step's gather reads
                                (step t - 1's, or step t's for an earlier layer in one-step mode), exactly as the
                                reference's compute(source.s) does.  Generic tier only, and not in a plan that also holds
                                an SNN_CONN_SPARSE connection or MCC features */
#define SNN_CONN_LOCAL2D 5 /* LocalConnection2D: per-target (unshared) receptive-field weights, topology.py:1623-1767.
                              Source [cin,hin,win], target n = cout * P neurons (cout = n_filters, P = hout * wout,
                              hout = (hin - kh) / sh + 1, wout likewise; ph = pw = 0, dh = dw = 1).  w is [cin, n, K]
                              with K = kh * kw; b is NULL.  Target n' = f * P + p (p = oy * wout + ox) receives
                                sum_ci ( sum_k s[ci, oy*sh + k / kw, ox*sw + k % kw] * w[ci, n', k] )
                              the inner sum over the spiking k ascending from +0, the outer one over ci ascending.
                              Rules SNN_RULE_NONE / NOOP / POSTPRE / WDEP_POSTPRE / HEBBIAN.  The rules' element
                              (n', m), m < cin * K, is flat weight n' * cin * K + m, and its source neuron is the one
                              at flat position (n' % P) * cin * K + m of the unfolded source in [cin, P, K] order (the
                              reference reshapes that view to [P, cin * K]; for cin = 1 it is the receptive field).
                              normalize: each row of w viewed as [cin * n, K] scaled by norm / (its sum, ascending k),
                              no guard against a zero sum.  Generic tier only, not with SNN_CONN_SPARSE or MCC features */
#define SNN_CONN_CONV3D 6  /* Conv3dConnection: F.conv3d(s.float(), w, b, stride, padding), topology.py:847-1025.
                              Source [cin,din,hin,win], target [cout,dout,hout,wout], both row-major; w is
                              [cout,cin,kd,kh,kw], b is [cout].  The conv fields keep the H and W axes (dh = dw = 1: the
                              reference refuses dilation); din, dout, kd, sd, pd (which share storage with the
                              SNN_CONN_SPARSE fields) the depth axis.  Each output size is (in - k + 2p) / s + 1 >= 1.
                              Target (co, oz, oy, ox) receives the sum of the taps whose zero-padded input position
                              spiked, in ascending (ci, kz, ky, kx) order from +0, then + b[co].  Rules: SNN_RULE_NONE,
                              SNN_RULE_NOOP (decay), and SNN_RULE_POSTPRE / WDEP_POSTPRE with nu0 = nu1 = 0 (decay, then
                              the clamp) — the reference's conv3d rules fail on any pre-synaptic term and pair the
                              post-synaptic one through transposed kernel axes, so a learning window with any other
                              rule is SNN_ERR_UNSUPPORTED.  normalize: each row of w viewed as [cout * cin, kd*kh*kw]
                              scaled by norm / (its sum, ascending), no guard against a zero sum.  No mask.  Generic
                              tier only, not with SNN_CONN_SPARSE or MCC features */
#define SNN_CONN_CONV1D 7  /* Conv1dConnection: F.conv1d(s.float(), w, b, stride, padding), topology.py:540-683.
                              Source [cin,win], target [cout,wout]; w is [cout,cin,kw], b is [cout].  The conv fields
                              with the height axis set to 1 (hin = hout = kh = sh = 1, ph = 0, dh = dw = 1);
                              wout = (win - kw + 2pw) / sw + 1 >= 1.  Target (co, ox) receives the sum of the taps whose
                              zero-padded input position spiked, in ascending (ci, kx) order from +0, then + b[co].
                              Rules SNN_RULE_NONE / NOOP / POSTPRE / WDEP_POSTPRE / HEBBIAN.  The rules' element (co, m),
                              m = ci * kw + kk < cin * kw, is flat weight co * cin * kw + m; it pairs target position l'
                              (L = wout) with the source neuron the reference's reshape of the unfolded source
                              [cin, L, kw] to [L, cin * kw] puts there: f = l' * cin * kw + m, c = f / (L * kw),
                              l = (f % (L * kw)) / kw, kk' = f % kw, source c * win + l * sw - pw + kk' (a padding
                              position: no term).  For cin = 1 this is the convolution's own pairing.
                                U = reduce_b sum_l' x_tgt[b, co, l'] * s_src[b, src],
                                V = reduce_b sum_l' s_tgt[b, co, l'] * x_src[b, src]
                              each sample's sum in ascending l', the samples' sums in ascending b, the terms of a silent
                              spike skipped; then PostPre / WeightDependentPostPre / Hebbian as on SNN_CONN_CONV2D,
                              decay and clamp.  normalize: each row of w viewed as [cout * cin, kw] scaled by
                              norm / (its sum, ascending), no guard against a zero sum.  No mask.  Generic tier only,
                              not with SNN_CONN_SPARSE or MCC features */
#define SNN_CONN_LOCAL3D 8 /* LocalConnection3D: per-target (unshared) receptive-field weights, topology.py:1770-1917.
                              The reference's source [cin, H, W, D] maps onto the conv fields with the innermost axis
                              kept contiguous: H -> din / kd / sd / dout (the depth fields SNN_CONN_CONV3D overlays on the
                              sparse storage), W -> hin / kh / sh / hout, D -> win / kw / sw / wout; so source neuron
                              (ci, z, y, x) is ((ci * din + z) * hin + y) * win + x.  Each output size is
                              (in - k) / s + 1 of a kernel that fits; pd = ph = pw = 0, dh = dw = 1; cout = n_filters.
                              w is [cin, n, K] with K = kd * kh * kw, k = (kz * kh + ky) * kw + kx (the reference's
                              flattening of its three unfolds); b is NULL.  Target n' = f * P + p, P = dout * hout * wout,
                              p = (oz * hout + oy) * wout + ox, receives
                                sum_ci ( sum_k s[ci, oz*sd + kz, oy*sh + ky, ox*sw + kx] * w[ci, n', k] )
                              the inner sum over the spiking k ascending from +0, the outer one over ci ascending.
                              Rules SNN_RULE_NONE / NOOP / POSTPRE / WDEP_POSTPRE / HEBBIAN, paired as on
                              SNN_CONN_LOCAL2D: element (n', m), m < cin * K, is flat weight n' * cin * K + m, and its
                              source neuron is the one at flat position (n' % P) * cin * K + m of the unfolded source in
                              [cin, P, K] order (for cin = 1 the receptive field).
                                U = reduce_b x_tgt[b, n'] * s_src[b, src],  V = reduce_b s_tgt[b, n'] * x_src[b, src]
                              the samples in ascending b from +0, the terms of a silent spike skipped; then the rule,
                              decay and clamp.  normalize: each row of w viewed as [cin * n, K] scaled by
                              norm / (its sum, ascending k), no guard against a zero sum.  No mask.  Generic tier only,
                              not with SNN_CONN_SPARSE, MCC features or per-neuron parameters; a library older than the
                              kind refuses it with SNN_ERR_UNSUPPORTED */
#define SNN_CONN_MAXPOOL3D 9 /* MaxPoo3dConnection: online-rate 3-D max pooling, topology.py:1214-1301.  No weights (w, b,
                                norm and mask absent), rule SNN_RULE_NOOP only.  Source [C,din,hin,win], target
                                [C,dout,hout,wout], both row-major: the H and W axes in the conv fields as on
                                SNN_CONN_MAXPOOL2D (cin = cout = C; kh/kw, sh/sw, ph/pw, dh/dw), the depth axis in
                                din, dout, kd, sd, pd, dd (the fields SNN_CONN_CONV3D overlays on the sparse storage),
                                each as for F.max_pool3d without ceil mode: padding at most half the kernel, and every
                                window holds an element of the volume on every axis.  Each compute:
                                  1. r = fl(r - fl(pool_decay * r)); r = fl(r + s)   on pool_rates [B,C,din,hin,win]
                                  2. idx = the first maximum of r[b,c] over the window in (kz, ky, kx) row-major order,
                                     padding never chosen (strict >, so -0 == +0 ties keep the earlier element; a NaN
                                     takes over)
                                  3. out[b,c,oz,oy,ox] = s[b,c,idx] as 0.0 / 1.0
                                The rates a step reads fold in the spikes that step's gather reads, as on
                                SNN_CONN_MAXPOOL2D.  Generic tier only; not in a plan that also holds an SNN_CONN_SPARSE
                                connection, MCC features or per-neuron parameters, and never into a PassThroughNodes
                                layer; a library older than the kind refuses it with SNN_ERR_UNSUPPORTED */
#define SNN_CONN_MEANFIELD 10 /* MeanFieldConnection: s.float().mean() * w, topology.py:1920-2006.  The mean runs over the
                                whole [B, n_src] spike tensor, the batch included, so every sample's input depends on
                                every sample's spikes:
                                  mean = fl((float)count / (float)(B * n_src)),  count = the number of spikes in s
                                  out[b, j] = fl(mean * w[mf_off[j] + b * mf_stride])
                                (exact while B * n_src < 2^24: the reference's CPU sum of 0 / 1 floats is the integer
                                count).  w is the connection's weight tensor in any shape that broadcasts into
                                [B, *target.shape] without growing it; mf_off [n_tgt] (int32) is the element of w target
                                neuron j of sample 0 reads, and mf_stride the step of a further sample (0 unless w has the
                                batch axis).  The result is added into the target's input at the connection's place in
                                the insertion order (network.py:244-248).  b is NULL; rule SNN_RULE_NOOP (w is never
                                written: learning.NoOp scales it by 1.0 and does not clamp) or SNN_RULE_NONE; no normalize,
                                no mask; the target is not a PassThroughNodes layer.  Every instantiation of the generic
                                kernel takes it; generic tier only (a forced tier 2 or 3 is SNN_ERR_UNSUPPORTED).  A
                                library older than the kind refuses it with SNN_ERR_UNSUPPORTED */
/* Weight normalisation with a per-target norm tensor, or after every step (MCC Weight(norm_frequency='time step'),
 * topology_features.py:633-671).  The flag is OR-ed into snn_conn_t.kind of an SNN_CONN_DENSE or SNN_CONN_MCC
 * connection with has_norm = 1; its norm_t / norm_step fields (they overlay the sparse storage) then describe the norm:
 *   norm_t     NULL: the scalar `norm`; else float32 [n_tgt], norm_t[j] is target j's norm
 *   norm_step  0: normalise at window end (normalize()), as without the flag;  1 (SNN_CONN_MCC only): normalise inside
 *              every compute instead, and never at window end
 * With S[j] = the column sum of w (|w| when norm_abs; summed in the SNN_NORM_CHUNKS order), S[j] == 0 -> 1:
 *   window end, scalar norm      f = fl(norm / S)            (unchanged)
 *   window end, norm_t           f = fl(norm_t[j] / S)       (Tensor / Tensor, topology.py:390-392, :264-266)
 *   per step, scalar norm        f = fl(fl(1 / S) * norm)    (float / Tensor is Tensor.__rtruediv__: reciprocal * norm)
 *   per step, norm_t             f = fl(norm_t[j] / S)
 * then w[i, j] = fl(w[i, j] * f).  Per step (norm_abs = 0: AbstractFeature.normalize sums the signed values), step t
 * gathers from w as step t - 1 left it, then normalises it, then the neurons update and the rule runs on the normalised
 * w (a clamping rule clamps every element, not only those its terms reach).  This holds with learning off, under
 * SNN_RULE_NONE and in one-step mode.  snn_b200_conn_normalize applies the formula the fields name (the per-step one
 * after a standalone compute); snn_b200_conn_compute and _update ignore the flag.  Generic tier only (tier 0 selects it, a forced tier 2 or 3 is
 * SNN_ERR_UNSUPPORTED); not with SNN_RULE_AVG, and not in a plan that also holds an SNN_CONN_SPARSE connection,
 * per-synapse tensors, per-neuron parameters or a kind of the pooling instantiation.  A library older than the flag
 * refuses such a plan with SNN_ERR_UNSUPPORTED (it rejects every kind above SNN_CONN_MEANFIELD). */
#define SNN_CONN_WNORM 0x100
#define SNN_RULE_NONE 0       /* MCC_learning.NoOp: update() does nothing    MCC_learning.py:120-146 */
#define SNN_RULE_NOOP 1        /* learning.NoOp: weight decay only, no clamp  learning.py:107-146     */
#define SNN_RULE_POSTPRE 2     /* learning.PostPre._connection_update         learning.py:390-420     */
#define SNN_RULE_WDEP_POSTPRE 3/* learning.WeightDependentPostPre             learning.py:626-653     */
#define SNN_RULE_MCC_POSTPRE 4 /* MCC_learning.PostPre._connection_update     MCC_learning.py:224-302 */
#define SNN_RULE_MSTDP 5       /* learning.MSTDP: reward-modulated STDP; _connection_update learning.py:1504-1574
                                  on SNN_CONN_DENSE, _conv2d_connection_update :1942-2015 on SNN_CONN_CONV2D;
                                  MCC_learning.MSTDP._connection_update MCC_learning.py:468-548 on SNN_CONN_MCC (the
                                  same arithmetic as on SNN_CONN_DENSE, with the same fields and pointers) */
#define SNN_RULE_HEBBIAN 6     /* learning.Hebbian: both terms positive, nu applied after the batch reduction;
                                  _connection_update learning.py:1110-1136, _conv2d_connection_update :1348-1380 */
/* On SNN_CONN_CONV2D the rules SNN_RULE_POSTPRE (learning.py:457-497), SNN_RULE_WDEP_POSTPRE (:920-975) and
 * SNN_RULE_HEBBIAN correlate the im2col views:  pre[co,k] = reduce_b sum_l x_tgt[b,co,l] * s_src_col[b,k,l],
 * post[co,k] = reduce_b sum_l s_tgt[b,co,l] * x_src_col[b,k,l]  (dilation 1), nu applied after the reduction. */
#define SNN_RULE_MSTDPET 7     /* learning.MSTDPET on a dense Connection (learning.py:2187-2249): reward-modulated STDP with an
                                  eligibility TRACE; batch size 1 only (the reference flattens the spikes of the whole batch into
                                  its [n] traces).  Also MCC_learning.MSTDPET (MCC_learning.py:652-733) on SNN_CONN_MCC, with the
                                  same fields and pointers as on SNN_CONN_DENSE */
#define SNN_RULE_IS_MSTDP(r) ((r) == SNN_RULE_MSTDP || (r) == SNN_RULE_MSTDPET)
/* MCC_learning.PostPre with average_update = k > 0 (MCC_learning.py:210-302): the flag is OR-ed into snn_conn_t.rule on
 * SNN_RULE_MCC_POSTPRE of an SNN_CONN_MCC connection, whose avg_* fields (they overlay the reward-rule state) then
 * describe the rule's averaging state, all updated in place:
 *   avg_pre / avg_post    float32 [k, n_src, n_tgt]: average_buffer_pre / _post
 *   avg_k                 k >= 1
 *   avg_idx_pre / _post   average_buffer_index_pre / _post, in [0, k): the slot the next update writes
 *   avg_continues         continues_update
 *   avg_rows              uint32 [k, ceil(n_src / 32)]: bit i of slot q set = row i of pre slot q may be non-zero
 *   avg_cols              uint32 [k, ceil(n_tgt / 32)]: bit j of slot q set = column j of post slot q may be non-zero
 *                         (all zero for zero buffers; a bit may be set over a row / column of zeros)
 * Each learning step, with U / V the step's batch-reduced terms of the plain rule without dt (s_src x fl(x_tgt * nu0) and
 * x_src x fl(s_tgt * nu1), samples ascending from +0, / B under SNN_REDUCE_MEAN):
 *   pre term, when nu0 != 0:  p = avg_idx_pre;  avg_pre[p] = U, avg_rows[p] = the rows with a spike in some sample;
 *                             avg_idx_pre = (p + 1) % k;  then, when avg_continues or avg_idx_pre == 0, every (i, j) with
 *                             row i set in some slot:  w = fl(w - fl(fl(S / k) * dt_scale)),  S = the sum of avg_pre[q][i][j]
 *                             over the slots q with row i set, q ascending from +0 (the mean over all k slots: the others
 *                             hold zeros, which leave such a sum as it is)
 *   post term, when nu1 != 0: the same with avg_post, avg_cols, columns, V and w = fl(w + ...)
 *   then decay and clamp as for the plain rule.  An element no applied term reaches keeps its value.
 * Nothing is touched for a zero rate, and nothing in a window with learning off.  Generic tier only (tier 0 selects it;
 * a forced tier 2 or 3 is SNN_ERR_UNSUPPORTED), no mask, and not in a plan that also holds an SNN_CONN_SPARSE connection,
 * per-synapse tensors, per-neuron parameters or a kind of the pooling instantiation.  A library older than the flag
 * refuses such a plan with SNN_ERR_UNSUPPORTED (it rejects every rule above SNN_RULE_MSTDPET). */
#define SNN_RULE_AVG 0x100
#define SNN_RULE_IS_STDP(r) (((r) >= SNN_RULE_POSTPRE && (r) <= SNN_RULE_MCC_POSTPRE) || (r) == SNN_RULE_HEBBIAN)

/* ---- broadcast forms of a dense connection's per-synapse tensors (snn_conn_t wmin_t / wmax_t / nu0_t / nu1_t): which
 *      element (i, j) of [n_src, n_tgt] reads ---- */
#define SNN_SYN_FULL 1 /* [n_src, n_tgt] row-major: t[i * n_tgt + j] */
#define SNN_SYN_TGT 2  /* per target neuron, [n_tgt] (or [1, n_tgt]): t[j] */
#define SNN_SYN_SRC 3  /* per source neuron, [n_src, 1]: t[i] */
#define SNN_SYN_ONE 4  /* one element: t[0] */

/* ---- weight-matrix structure hints (DiehlAndCook2015's static exc/inh matrices,
 *      models.py:204,217-220) ---- */
#define SNN_W_DENSE 0   /* arbitrary dense matrix                                              */
#define SNN_W_DIAG 1    /* square, w[i][i] = structure_val, 0 elsewhere                        */
#define SNN_W_OFFDIAG 2 /* square, w[i][i] = 0, structure_val elsewhere                        */

/* ---- batch reduction of the STDP update (learning.py:76-80) ---- */
#define SNN_REDUCE_SUM 0  /* torch.sum; also torch.squeeze when B == 1 */
#define SNN_REDUCE_MEAN 1 /* torch.mean */

/* ---- external input dtype ---- */
#define SNN_EXT_NONE 0
#define SNN_EXT_U8 1  /* uint8 / bool, one byte per element */
#define SNN_EXT_F32 2 /* float32 */

/* ---- status codes (snn_*_run_window return value and *err_flag bits) ---- */
#define SNN_OK 0
#define SNN_ERR_BAD_ARG 1        /* malformed plan (sizes, indices, NULLs)                        */
#define SNN_ERR_UNSUPPORTED 2    /* valid reference configuration this build does not implement   */
#define SNN_ERR_WORKSPACE 4      /* workspace too small                                           */
#define SNN_ERR_CUDA 8           /* a CUDA runtime call failed                                    */
#define SNN_ERR_NONBINARY 16     /* (device flag) an Input layer received, or an SNN_NODE_PASSTHROUGH layer held or
                                    received, a value outside {0,1} (spikes are carried as bits)    */
#define SNN_ERR_BARRIER 32       /* (device flag) grid barrier timed out — kernel bailed out      */
#define SNN_ERR_STRUCTURE 64     /* (device flag) a weight matrix does not have the structure its SNN_W_* hint claims */

/* One population of neurons.  Reference: Nodes.__init__ nodes.py:15-86 + subclass ctor. */
typedef struct snn_layer {
    int32_t kind;            /* SNN_NODE_*                                                 */
    int32_t n;               /* neurons per sample                                         */
    int32_t traces;          /* Nodes.traces                                               */
    int32_t traces_additive; /* Nodes.traces_additive                                      */
    int32_t sum_input;       /* Nodes.sum_input                                            */
    int32_t learning;        /* layer.learning (gates theta adaptation, nodes.py:1078,1093) */
    int32_t one_spike;       /* DiehlAndCookNodes.one_spike (nodes.py:1097-1105)            */
    int32_t has_lbound;      /* lbound is not None                                         */
    float dt;                /* layer.dt (nodes.py:127)                                    */
    float trace_decay;       /* exp(-dt/tc_trace), evaluated in fp32 like nodes.py:129-131 */
    float trace_scale;
    float decay;             /* exp(-dt/tc_decay)  nodes.py:546-548,1128-1130              */
    float rest, reset, thresh, refrac, lbound;
    float theta_plus;        /* DC only */
    float theta_decay;       /* DC only: exp(-dt/tc_theta_decay) nodes.py:1131-1133        */
    int32_t ext_dtype;       /* SNN_EXT_*: dtype of `ext`                                  */
    int32_t clamp_per_step;  /* 0: clamp is [n]; 1: clamp is [T,n]   (network.py:416-421)   */
    int32_t unclamp_per_step;
    int32_t inject_per_step;
    /* --- state, updated in place; shapes as in the reference --- */
    uint8_t *s;          /* [B,n] 0/1.  in: spikes of step -1, out: spikes of step T-1      
                            (SNN_NODE_PASSTHROUGH: float32 0.0 / 1.0)                         */
    float *v;            /* [B,n]  (LIF, DC)                                                */
    float *refrac_count; /* [B,n]  (LIF, DC)                                                */
    float *x;            /* [B,n]  if traces                                                */
    float *theta;        /* [n]    (DC) — shared across the batch, nodes.py:1061            */
    float *summed;       /* [B,n]  if sum_input                                             */
    /* --- per-window inputs --- */
    const void *ext;        /* [T,B,n] external input (network.py:388-392) or NULL          */
    const uint8_t *clamp;   /* bool mask, force s=1 after forward (network.py:415-421)      */
    const uint8_t *unclamp; /* bool mask, force s=0 after forward (network.py:423-429)      */
    const float *inject_v;  /* added to v before forward (network.py:398-404)               */
    /* --- per-window recordings (Monitor, monitors.py:94-111); NULL = not recorded --- */
    uint8_t *rec_s; /* [T,B,n] */
    float *rec_v;   /* [T,B,n] */
    int32_t *rec_count; /* [B,n] += number of spikes of each neuron over the window (what the
                           reference's callers compute as spikes.sum(time), e.g.
                           examples/mnist/batch_eth_mnist.py:280-284); NULL = not counted */
    /* SNN_NODE_CURRENT_LIF: the synaptic current.  An SNN_NODE_LIF / SNN_NODE_DC layer never reads these fields, so the
       same storage carries its per-neuron parameter block when its kind has the SNN_NODE_PN flag (see there). */
    union {
        struct {
            float *i;           /* [B,n] synaptic input current, updated in place (nodes.py:771,778) */
            float i_decay;      /* exp(-dt/tc_i_decay) (nodes.py:818-820) */
        };
        struct {
            const float *pn;    /* SNN_NODE_PN: float32 [k, n], row r = the SNN_PN_* parameter r of every neuron */
            uint32_t pn_mask;   /* SNN_NODE_PN: bit r set = row r replaces the scalar field of parameter r */
        };
    };
} snn_layer_t;

/* One dense synapse matrix.  Reference: Connection (topology.py:265-399) or
 * MulticompartmentConnection with a single Weight feature (topology.py:402-537,
 * topology_features.py:575-671). */
typedef struct snn_conn {
    int32_t kind;      /* SNN_CONN_*                                                        */
    int32_t src, tgt;  /* indices into layers[]                                             */
    int32_t rule;      /* SNN_RULE_*                                                        */
    int32_t reduction; /* SNN_REDUCE_*                                                      */
    int32_t has_norm;  /* normalize at window end (network.py:464-465)                      */
    int32_t norm_abs;  /* 1: divide by sum_i |w| (topology.py:390-392); 0: plain sum
                          (topology_features.py:264-266)                                    */
    int32_t has_clamp; /* rule clamps w to [wmin,wmax] after each update (learning.py:97-104,
                          MCC_learning.py:101-110)                                          */
    int32_t structure; /* SNN_W_*: caller-verified structure of w (plan-time hint that lets the
                          fused kernel skip a static n x n matrix; SNN_W_DENSE is always valid) */
    float nu0, nu1;    /* pre-/post-synaptic learning rates                                 */
    float wmin, wmax;
    float weight_decay;/* multiplicative per-step factor (learning.py:85,93-94); 1.0 = off  */
    float dt_scale;    /* MCC: connection.dt factor on both STDP terms (MCC_learning.py:262,298) */
    float norm;
    float structure_val; /* the constant of SNN_W_DIAG / SNN_W_OFFDIAG                      */
    float *w;          /* [n_src, n_tgt] row-major, updated in place (CONV2D: [Cout,Cin,kh,kw]) */
    const float *b;    /* [n_tgt] bias or NULL (topology.py:345); CONV2D: [Cout]            */
    /* SNN_CONN_CONV2D geometry (topology.py:738-760): source [cin,hin,win], target [cout,hout,wout] */
    int32_t cin, hin, win, cout, hout, wout, kh, kw, sh, sw, ph, pw, dh, dw;
    /* SNN_RULE_MSTDP (learning.py:1440-1574, 1942-2015; MCC_learning.py:392-551).  State of the rule, updated in place:
         DENSE, MCC: p_plus [B,n_src], p_minus [B,n_tgt]; the eligibility [B,n_src,n_tgt] of the previous
                 step is NOT materialised: it is p_plus (x) s_post + s_pre (x) p_minus of that step, so
                 the spikes the rule saw last are kept instead (mst_spre [B,n_src], mst_spost [B,n_tgt],
                 one byte per neuron);
         CONV2D: p_plus is the [B,cin,hin,win] trace image whose im2col the reference stores
                 (unfold is linear), p_minus [B,cout*hout*wout], elig [B,cout,cin*kh*kw] (fp32,
                 materialised like the reference's, applied one step later).                  */
    /* SNN_RULE_MCC_POSTPRE | SNN_RULE_AVG keeps its averaging state in the same storage (see there): a connection never
       has both rules, so the layout is the one without it. */
    union {
        struct {
            float reward;      /* the run's scalar reward (network.py:319-377 -> kwargs["reward"])  */
            float a_plus, a_minus;           /* defaults +1 / -1 (learning.py:1543-1556)            */
            float p_plus_decay, p_minus_decay; /* exp(-dt/tc_plus), exp(-dt/tc_minus), computed by the host in fp32 */
            float *p_plus, *p_minus, *elig;
            uint8_t *mst_spre, *mst_spost;
        };
        struct {
            float *avg_pre, *avg_post;
            uint32_t *avg_rows, *avg_cols;
            int32_t avg_k, avg_idx_pre, avg_idx_post, avg_continues;
        };
    };
    /* Network.run(..., masks={(source, target): mask}) (network.py:279-280,321,449): weights whose mask byte is non-zero are
       forced to 0 after every step's update, learning or not (AbstractConnection.update, topology.py:127-131).  [n_src, n_tgt]
       bytes, SNN_CONN_DENSE only (MulticompartmentConnection.update ignores the kwarg, topology.py:509-518); NULL = none. */
    const uint8_t *mask;
    /* SNN_RULE_MSTDPET (learning.py:2187-2249; MCC_learning.py:554-738), SNN_CONN_DENSE or SNN_CONN_MCC, B = 1.  p_plus [n_src], p_minus [n_tgt], mst_spre / mst_spost as for
       SNN_RULE_MSTDP (the eligibility of the previous step is rebuilt from them); e_trace [n_src, n_tgt] is the rule's
       eligibility_trace, updated in place:  e_trace = e_trace * e_trace_decay + eligibility / tc_e_trace  (:2229-2230),
       w += et_coef * e_trace  with et_coef = nu[0] * dt * reward evaluated by the host in fp32 (:2232-2238). */
    float *e_trace;
    float e_trace_decay, tc_e_trace, et_coef;
    /* SNN_CONN_SPARSE: compressed sparse rows of the [n_src, n_tgt] pattern.  sp_rowptr [n_src + 1], monotone, in
       [0, nnz]; sp_col [nnz], strictly ascending within a row, < n_tgt; w [nnz] the values in the same order, decayed
       in place by SNN_RULE_NOOP.  A malformed pattern is reported as SNN_ERR_BAD_ARG (in *err_flag by the window).
       SNN_CONN_CONV3D (topology.py:847-1025) keeps its depth axis in the same storage: source depth din, target depth
       dout, kernel depth kd, stride sd, padding pd; SNN_CONN_MAXPOOL3D also its depth dilation dd (read by no other
       kind).  SNN_CONN_MEANFIELD keeps its offset map and per-sample stride there, and an SNN_CONN_DENSE or
       SNN_CONN_MCC connection with SNN_CONN_WNORM its norm tensor and per-step flag.  A connection is never two of these
       kinds, so the layout is the one without them. */
    union {
        struct {
            const int32_t *sp_rowptr;
            const int32_t *sp_col;
            int32_t nnz;
        };
        struct {
            int32_t din, dout, kd, sd, pd, dd;
        };
        struct {
            const int32_t *mf_off;   /* SNN_CONN_MEANFIELD: [n_tgt] element of w per target neuron (sample 0) */
            int32_t mf_stride;       /* SNN_CONN_MEANFIELD: elements of w between consecutive samples (0: shared) */
        };
        struct {
            const float *norm_t;     /* SNN_CONN_WNORM: float32 [n_tgt] per-target norm, NULL = the scalar norm */
            int32_t norm_step;       /* SNN_CONN_WNORM: 1 = normalise after every step's compute (SNN_CONN_MCC) */
        };
    };
    /* SNN_CONN_MCC with Probability / Mask / Intensity features besides its Weight (topology.py:437-479).  Each is an
       [n_src, n_tgt] row-major matrix or NULL (feature absent).  A spiking source i adds fl(w[i,j] * f_int[i,j]) (just
       w[i,j] without f_int) to target j when f_mask[i,j] != 0 and the Probability draw of synapse (i, j) transmits
       (snn_synapse_transmits with f_prob[i,j]); otherwise it adds nothing.  The sum is the plain MCC gather's: i
       ascending, from +0.  The draw is one [n_src, n_tgt] mask per step, shared by every sample of the batch
       (torch.bernoulli(value) broadcast over B, topology_features.py:425-429).  The window draws with (opts.seed,
       opts.step_offset + t, connection index); snn_b200_conn_compute with (draw_seed, draw_step, draw_conn).  Generic
       tier only, and not in a plan that also holds an SNN_CONN_SPARSE connection. */
    /* SNN_CONN_DENSE keeps its per-synapse tensors in the same storage (a connection is never both kinds): wmin_t / wmax_t
       are AbstractConnection.wmin / wmax (topology.py:74-81) and nu0_t / nu1_t the rows of LearningRule.nu =
       torch.stack(nu) (learning.py:58-67), each float32 in the broadcast form its *_form byte names (SNN_SYN_*).  NULL
       = the scalar field (wmin, wmax, nu0, nu1) holds the value.  nu0_t and nu1_t are set together.  Where a tensor is
       set, the element (i, j) takes the scalar's place in every formula of the connection's rule:
         clamp           w = clamp(w, wmin[i,j], wmax[i,j])  every step, for every rule but NOOP (has_clamp as for scalars:
                         some element of wmin is not -inf, or some element of wmax is not +inf; learning.py:97-104)
         POSTPRE         nu broadcast to [1, n_tgt] only (SNN_SYN_TGT / SNN_SYN_ONE; any other form is the reference's
                         bmm shape error, SNN_ERR_BAD_ARG): U sums s_src * fl(x_tgt * nu0[j]), V sums x_src * nu1[j]
         WDEP_POSTPRE    upd = 0 - fl(fl(nu0[i,j] * U) * (w - wmin[i,j])) + fl(fl(nu1[i,j] * V) * (wmax[i,j] - w))
         HEBBIAN         w = w + nu0[i,j] * U;  w = w + nu1[i,j] * V
         MSTDP           w = w + nu0[i,j] * upd
         MSTDPET         w = w + fl(fl(fl(nu0[i,j] * dt_scale) * reward) * e_trace), dt_scale = connection.dt (et_coef unused)
       With nu tensors the scalars nu0 / nu1 are the rule's gates: 0 when nu[k].any() is false, otherwise any non-zero
       value (HEBBIAN applies its rates without a gate: nu0 = nu1 = 1).  Generic tier only (tier 0 selects it, a forced tier
       2 or 3 is SNN_ERR_UNSUPPORTED), and not in a plan that also holds an SNN_CONN_SPARSE connection, MCC features or a
       kind of the pooling instantiation.  A library older than these fields refuses such a plan (wmin_t, wmax_t and
       nu0_t overlay f_prob / f_mask / f_int, which it accepts on SNN_CONN_MCC only). */
    union {
        struct {
            const float *f_prob;    /* Probability.value, each in [0, 1]                    topology_features.py:365-464 */
            const uint8_t *f_mask;  /* Mask.value, 0 / 1 bytes                              topology_features.py:467-549 */
            const float *f_int;     /* Intensity.value                                      topology_features.py:724-769 */
            uint32_t draw_seed, draw_step, draw_conn;
        };
        struct {
            const float *wmin_t, *wmax_t, *nu0_t, *nu1_t;
            int8_t wmin_form, wmax_form, nu0_form, nu1_form;
        };
    };
    /* SNN_CONN_MAXPOOL2D (topology.py:1124-1211) and SNN_CONN_MAXPOOL3D (:1214-1301): the firing_rates buffer
       [B, C, hin, win] (3-D: [B, C, din, hin, win]), updated in place (after a
       window it holds what the reference's buffer holds after the window's last compute), and the decay kwarg rounded
       to fp32 as `decay * firing_rates` rounds it. */
    float *pool_rates;
    float pool_decay;
} snn_conn_t;

typedef struct snn_net {
    int32_t abi_version; /* SNN_ABI_VERSION */
    int32_t n_layers;
    int32_t n_conns;
    int32_t learning;    /* network.learning: gates connection.update() (network.py:448-450) */
    snn_layer_t layers[SNN_MAX_LAYERS];
    snn_conn_t conns[SNN_MAX_CONNS];
} snn_net_t;

typedef struct snn_run_opts {
    int32_t T;             /* timesteps = int(time / dt)  (network.py:356)                    */
    int32_t B;             /* batch size                                                      */
    int32_t normalize;     /* 1: run every connection's normalize() after the loop            */
    int32_t tier;          /* 0 = auto (fused v1 where it matches, else fused v2, else generic), 1 = force generic kernel,
                              2 = force fused DC2015 kernel v1 (grid barrier), 3 = force fused DC2015 kernel v2
                              (exchange warp, per-column-group pipelines) */
    uint32_t seed;         /* one_spike tie-break stream (see snn_one_spike_key)              */
    uint32_t step_offset;  /* added to t in the tie-break hash (lets callers split a window)  */
    int32_t *err_flag;     /* optional int32 (device memory for the CUDA lib); OR-ed with SNN_ERR_* */
    int32_t one_step;  /* Network.run(one_step=True), network.py:383-396: each layer's input is recomputed from
                          the CURRENT spikes of its sources just before its forward (generic tier only) */
    /* Multi-GPU windows (SURVEY.md section 8e; the reference has no counterpart).  When delta_w / delta_theta are set
     * the window leaves the learned weights / adaptive thresholds of the DiehlAndCook2015 graph as they were at the
     * start and writes what it would have added instead — delta_w[i*n+j] = w_end - w_start, delta_theta[j] =
     * theta_end - theta_start — straight into the caller's all-reduce buffer (no snapshot, no separate subtraction
     * pass).  Fused DC2015 kernel (tier 2) only, normalize must be 0; anything else: SNN_ERR_UNSUPPORTED. */
    float *delta_w;
    float *delta_theta;
} snn_run_opts_t;

/*
 * one_spike tie-break.  The reference draws the single winner per sample with
 * torch.multinomial over the 0/1 candidate mask (nodes.py:1097-1105), i.e. uniformly among
 * the threshold crossers.  We draw it as the arg-max over the candidates of an i.i.d. 31-bit
 * hash of (seed, step, layer, sample, neuron) — the same distribution, but computable with one
 * atomicMax per sample across the whole grid.  The key packs the hash above the neuron index so
 * that the arg-max also returns the winner.  The oracle and the golden generator (which
 * monkey-patches torch.multinomial with it) use this very definition.
 */
#ifdef __CUDACC__
#define SNN_HD __host__ __device__
#else
#define SNN_HD
#endif
static inline SNN_HD uint32_t snn_fmix32(uint32_t h) {
    h ^= h >> 16; h *= 0x85EBCA6Bu; h ^= h >> 13; h *= 0xC2B2AE35u; h ^= h >> 16; return h;
}
static inline SNN_HD uint32_t snn_one_spike_hash(uint32_t seed, uint32_t t, uint32_t layer, uint32_t b, uint32_t j) {
    uint32_t h = snn_fmix32(seed ^ (0x9E3779B9u * (t + 1u)));
    h = snn_fmix32(h + 0x85EBCA6Bu * (layer + 1u) + b);
    h = snn_fmix32(h ^ (0xC2B2AE35u * (j + 1u)));
    return h;
}
static inline SNN_HD uint64_t snn_one_spike_key(uint32_t seed, uint32_t t, uint32_t layer, uint32_t b, uint32_t j) {
    return ((uint64_t)(snn_one_spike_hash(seed, t, layer, b, j) | 0x80000000u) << 32) | (uint64_t)j;
}

/*
 * Probability feature draw.  The reference transmits synapse (i, j) with torch.bernoulli(value): one [n_src, n_tgt]
 * draw per MulticompartmentConnection.compute call, i.e. per step, broadcast over the batch (topology_features.py:
 * 425-429).  We draw it from a counter-based 32-bit hash of (seed, step, connection, i, j): the source row is hashed
 * once (snn_synapse_row), each column then costs one mixing round (snn_synapse_col).  The leading tag 0x53594E41
 * keeps this stream apart from snn_one_spike_hash even under the same seed.  The synapse transmits when
 * (h >> 8) * 2^-24 < p, exact in fp32: p = 0 never transmits, p = 1 always does.  The oracle, the kernels and the
 * golden generator (which patches the reference's Probability.compute with it) share this definition.
 */
static inline SNN_HD uint32_t snn_synapse_row(uint32_t seed, uint32_t t, uint32_t conn, uint32_t i) {
    uint32_t h = snn_fmix32(seed ^ 0x53594E41u);
    h = snn_fmix32(h ^ (0x9E3779B9u * (t + 1u)));
    h = snn_fmix32(h ^ (0x85EBCA6Bu * (conn + 1u)));
    return snn_fmix32(h ^ (0xC2B2AE35u * (i + 1u)));
}
static inline SNN_HD uint32_t snn_synapse_col(uint32_t row, uint32_t j) { return snn_fmix32(row ^ (0x27D4EB2Fu * (j + 1u))); }
static inline SNN_HD uint32_t snn_synapse_draw(uint32_t seed, uint32_t t, uint32_t conn, uint32_t i, uint32_t j) {
    return snn_synapse_col(snn_synapse_row(seed, t, conn, i), j);
}
static inline SNN_HD int snn_synapse_transmits(uint32_t h, float p) { return (float)(h >> 8) * 5.9604644775390625e-08f < p; }

/* Row-chunking of the end-of-window column sum (normalize): rows are split into
 * SNN_NORM_CHUNKS contiguous chunks of ceil(n_src/SNN_NORM_CHUNKS) rows, each summed in
 * ascending row order, and the partial sums are then added in ascending chunk order.  Both
 * libraries use this fixed order so that their results are bit-identical. */
#define SNN_NORM_CHUNKS 16

/* ------------------------------------------------------------------------------------------
 * CUDA library (libsnn_b200.so).  Every pointer inside `net`/`opts` is a device pointer on the
 * current device; `stream` is a cudaStream_t (NULL = legacy default stream).  Calls are
 * asynchronous with respect to the host; no host synchronisation happens inside.
 * ------------------------------------------------------------------------------------------ */

/* Bytes of scratch the window needs (spike bitmaps, tie-break keys, barrier words).
 * Replaces: the per-step temporaries the reference allocates inside Network.run
 * (network.py:240-242; topology.py:454; MCC_learning.py:234-299). */
size_t snn_b200_workspace_bytes(const snn_net_t *net, const snn_run_opts_t *opts);

/* Run one window.  Replaces: Network.run's timestep loop + end-of-run normalize
 * (network.py:380-465) together with everything it dispatches to: _get_inputs
 * (network.py:211-250), Nodes.forward (nodes.py:96-107,211-221,500-529,1069-1111),
 * Connection.compute / MulticompartmentConnection.compute (topology.py:332-346,437-479),
 * LearningRule.update (learning.py:87-104,390-420,626-653; MCC_learning.py:86-110,224-302),
 * Monitor.record (monitors.py:94-111) and normalize (topology.py:383-392;
 * topology_features.py:250-266).  Returns SNN_OK or an SNN_ERR_* code (host-detectable
 * errors only; device-detected errors are OR-ed into *opts->err_flag). */
int snn_b200_run_window(const snn_net_t *net, const snn_run_opts_t *opts, void *workspace,
                        size_t workspace_bytes, void *stream);

/* Which kernel tier `tier = 0` would select for this plan: 1 generic, 2 fused DC2015 (v1), 3 fused DC2015 (v2). */
int snn_b200_select_tier(const snn_net_t *net, const snn_run_opts_t *opts);

/* Number of kernel launches the last snn_b200_run_window on this thread issued. */
int snn_b200_last_launch_count(void);

/* Multi-GPU window combine (no reference equivalent: SURVEY.md §8e).  After an
 * all-reduce(sum) of dw = w_local - w0 over ranks:  w = clamp(w0 + dw_sum, wmin, wmax),
 * then, if has_norm, the column normalisation of normalize().  n_src x n_tgt row-major. */
int snn_b200_delta_prepare(const float *w, const float *w0, float *dw, size_t count, void *stream);
int snn_b200_delta_apply(float *w, const float *w0, const float *dw_sum, int32_t n_src, int32_t n_tgt,
                         int32_t has_clamp, float wmin, float wmax, int32_t has_norm, int32_t norm_abs,
                         float norm, void *stream);
/* The same combine in place for a window run with snn_run_opts_t.delta_w / delta_theta (w still holds the weights of
 * the window start): w = clamp(w + dw_sum), normalize(), theta = theta + dtheta_sum — one launch.  theta may be NULL. */
int snn_b200_delta_apply_fused(float *w, const float *dw_sum, int32_t n_src, int32_t n_tgt, int32_t has_clamp, float wmin, float wmax,
                               int32_t has_norm, int32_t norm_abs, float norm, float *theta, const float *dtheta_sum, int32_t n_theta,
                               void *stream);

/* Single-operator entry points — the reference's per-object methods, for callers that drive
 * the objects themselves instead of through Network.run:
 *   snn_b200_conn_compute   = Connection.compute / MulticompartmentConnection.compute
 *                             (topology.py:332-346,437-479): out[b,j] = sum_i s[b,i] w[i,j] (+ b[j])
 *   snn_b200_conn_update    = connection.update(learning=True) for conns[conn_index] from the
 *                             layers' CURRENT s / x (topology.py:112-139, learning.py:87-104,390-420,
 *                             626-653; MCC_learning.py:86-110,224-302)
 *   snn_b200_conn_normalize = Connection.normalize / AbstractFeature.normalize
 *                             (topology.py:383-392, topology_features.py:250-266) */
int snn_b200_conn_compute(const snn_conn_t *conn, int32_t n_src, int32_t n_tgt, int32_t B, const uint8_t *s,
                          float *out, void *stream);
int snn_b200_conn_update(const snn_net_t *net, int32_t conn_index, int32_t B, void *workspace,
                         size_t workspace_bytes, void *stream);
int snn_b200_conn_normalize(const snn_conn_t *conn, int32_t n_src, int32_t n_tgt, void *stream);

/* On-device spike encoders — the step before the hot path (SURVEY.md §8f rank 1): the reference's callers encode on
 * the CPU and ship [time, batch, ...] uint8 spikes to the device; these write the same tensor on the device from the
 * rate image.  `out` is [T][n] uint8 (n = batch * pixels, the element order of the rate tensor), 0/1.
 *   snn_b200_encode_poisson   = bindsnet.encoding.poisson (encodings.py:99-156): rate_hz[n] in Hz, inter-spike intervals
 *                               ~ Poisson(1000 / (rate * dt)) steps, zero intervals bumped to one, rate 0 never spikes
 *   snn_b200_encode_bernoulli = bindsnet.encoding.bernoulli (encodings.py:50-96): prob[n] = max_prob * normalised datum,
 *                               one independent trial per step
 * Counter-based Philox-4x32-10 keyed by (seed, element): same distribution as the reference, not its random stream. */
int snn_b200_encode_poisson(const float *rate_hz, int32_t n, int32_t T, float dt, uint64_t seed, uint8_t *out, void *stream);
int snn_b200_encode_bernoulli(const float *prob, int32_t n, int32_t T, uint64_t seed, uint8_t *out, void *stream);

/* Label assignment and classification from per-sample spike counts — the step after the hot path (SURVEY.md §8f rank 2).
 * `counts` is [n_samples, n_neurons] int32: what snn_layer_t.rec_count accumulates over a window, i.e. the reference's
 * `spikes.sum(1)` (evaluation.py:41,115,160) without the [n_samples, time, n_neurons] raster.
 *   snn_b200_assign_labels = bindsnet.evaluation.assign_labels (evaluation/evaluation.py:8-61): rates [n, L] updated in
 *                            place (alpha-decayed running per-class mean counts), proportions [n, L], assignments [n] (int64)
 *   snn_b200_predict       = all_activity (evaluation.py:99-136; proportions == NULL) / proportion_weighting (:139-180):
 *                            predictions [n_samples] int64 */
int snn_b200_assign_labels(const int32_t *counts, const int64_t *labels, int32_t n_samples, int32_t n_neurons, int32_t n_labels, float alpha,
                           float *rates, float *proportions, int64_t *assignments, void *stream);
int snn_b200_predict(const int32_t *counts, const int64_t *assignments, const float *proportions, int32_t n_samples, int32_t n_neurons,
                     int32_t n_labels, int64_t *predictions, void *stream);

/* Library/ABI identification. */
int snn_b200_abi_version(void);
const char *snn_b200_build_info(void);

/* ------------------------------------------------------------------------------------------
 * Oracle library (libsnn_oracle.so) — TEST INFRASTRUCTURE, host pointers, never shipped on the
 * product path.  `dense` = 1 evaluates every product of the reference's dense formulation
 * (zeros included, like `s.float() @ w` and the batch-summed outer products); 0 skips
 * exact-zero terms.  Both give bit-identical results.  `threads` <= 0 means all cores.
 * ------------------------------------------------------------------------------------------ */
int snn_oracle_run_window(const snn_net_t *net, const snn_run_opts_t *opts, int dense, int threads);
int snn_oracle_delta_apply(float *w, const float *w0, const float *dw_sum, int32_t n_src, int32_t n_tgt,
                           int32_t has_clamp, float wmin, float wmax, int32_t has_norm, int32_t norm_abs,
                           float norm);
int snn_oracle_conn_compute(const snn_conn_t *conn, int32_t n_src, int32_t n_tgt, int32_t B, const uint8_t *s,
                            float *out);
int snn_oracle_conn_update(const snn_net_t *net, int32_t conn_index, int32_t B);
int snn_oracle_conn_normalize(const snn_conn_t *conn, int32_t n_src, int32_t n_tgt);
int snn_oracle_abi_version(void);

#ifdef __cplusplus
}
#endif
#endif /* SNN_B200_H */
