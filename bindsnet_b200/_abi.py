"""ctypes mirror of ``include/snn_b200.h`` (the C ABI of the simulation core).

The structs here must match the header field for field; ``tests/test_abi.py`` checks the
sizes against the values the compiled libraries report and that every symbol the header
declares is exported.
"""
from __future__ import annotations

import ctypes as C

SNN_ABI_VERSION = 13
SNN_MAX_LAYERS = 8
SNN_MAX_CONNS = 12

SNN_NODE_INPUT, SNN_NODE_LIF, SNN_NODE_DC, SNN_NODE_IF, SNN_NODE_CURRENT_LIF, SNN_NODE_BOOSTED_LIF, SNN_NODE_MCP = 0, 1, 2, 3, 4, 5, 6
SNN_NODE_SUBIF, SNN_NODE_PASSTHROUGH = 7, 8
SNN_CONN_DENSE, SNN_CONN_MCC, SNN_CONN_CONV2D, SNN_CONN_SPARSE, SNN_CONN_MAXPOOL2D, SNN_CONN_LOCAL2D = 0, 1, 2, 3, 4, 5
SNN_CONN_CONV3D, SNN_CONN_CONV1D, SNN_CONN_LOCAL3D, SNN_CONN_MAXPOOL3D, SNN_CONN_MEANFIELD = 6, 7, 8, 9, 10
SNN_CONN_WNORM = 0x100
SNN_RULE_NONE, SNN_RULE_NOOP, SNN_RULE_POSTPRE, SNN_RULE_WDEP_POSTPRE, SNN_RULE_MCC_POSTPRE, SNN_RULE_MSTDP, SNN_RULE_HEBBIAN = 0, 1, 2, 3, 4, 5, 6
SNN_RULE_MSTDPET = 7
SNN_RULE_AVG = 0x100
SNN_REDUCE_SUM, SNN_REDUCE_MEAN = 0, 1
SNN_EXT_NONE, SNN_EXT_U8, SNN_EXT_F32 = 0, 1, 2
SNN_W_DENSE, SNN_W_DIAG, SNN_W_OFFDIAG = 0, 1, 2
SNN_SYN_FULL, SNN_SYN_TGT, SNN_SYN_SRC, SNN_SYN_ONE = 1, 2, 3, 4
SNN_NODE_PN = 0x100
(SNN_PN_THRESH, SNN_PN_REST, SNN_PN_DECAY, SNN_PN_THETA_PLUS, SNN_PN_THETA_DECAY, SNN_PN_TRACE_DECAY,
 SNN_PN_TRACE_SCALE) = range(7)
SNN_PN_ROWS = 7

SNN_OK = 0
SNN_ERR_BAD_ARG = 1
SNN_ERR_UNSUPPORTED = 2
SNN_ERR_WORKSPACE = 4
SNN_ERR_CUDA = 8
SNN_ERR_NONBINARY = 16
SNN_ERR_BARRIER = 32
SNN_ERR_STRUCTURE = 64

ERR_NAMES = {
    SNN_ERR_BAD_ARG: "malformed plan",
    SNN_ERR_UNSUPPORTED: "configuration not implemented by the CUDA core",
    SNN_ERR_WORKSPACE: "workspace too small",
    SNN_ERR_CUDA: "CUDA runtime error",
    SNN_ERR_NONBINARY: "Input layer received, or PassThroughNodes layer held or received, values outside {0,1}",
    SNN_ERR_BARRIER: "grid barrier timed out",
    SNN_ERR_STRUCTURE: "a static weight matrix no longer has the diagonal / constant off-diagonal structure it was planned with",
}


def describe_error(code: int) -> str:
    return ", ".join(name for bit, name in ERR_NAMES.items() if code & bit) or f"status {code}"


class _CurrentFields(C.Structure):
    _fields_ = [("i", C.c_void_p), ("i_decay", C.c_float)]


class _NeuronParamFields(C.Structure):
    _fields_ = [("pn", C.c_void_p), ("pn_mask", C.c_uint32)]


class _CurrentOrNeuronParams(C.Union):
    """The storage SNN_NODE_CURRENT_LIF's current and an SNN_NODE_PN layer's per-neuron block share."""

    _anonymous_ = ("_cur", "_pn")
    _fields_ = [("_cur", _CurrentFields), ("_pn", _NeuronParamFields)]


class SnnLayer(C.Structure):
    _anonymous_ = ("_u",)
    _fields_ = [
        ("kind", C.c_int32),
        ("n", C.c_int32),
        ("traces", C.c_int32),
        ("traces_additive", C.c_int32),
        ("sum_input", C.c_int32),
        ("learning", C.c_int32),
        ("one_spike", C.c_int32),
        ("has_lbound", C.c_int32),
        ("dt", C.c_float),
        ("trace_decay", C.c_float),
        ("trace_scale", C.c_float),
        ("decay", C.c_float),
        ("rest", C.c_float),
        ("reset", C.c_float),
        ("thresh", C.c_float),
        ("refrac", C.c_float),
        ("lbound", C.c_float),
        ("theta_plus", C.c_float),
        ("theta_decay", C.c_float),
        ("ext_dtype", C.c_int32),
        ("clamp_per_step", C.c_int32),
        ("unclamp_per_step", C.c_int32),
        ("inject_per_step", C.c_int32),
        ("s", C.c_void_p),
        ("v", C.c_void_p),
        ("refrac_count", C.c_void_p),
        ("x", C.c_void_p),
        ("theta", C.c_void_p),
        ("summed", C.c_void_p),
        ("ext", C.c_void_p),
        ("clamp", C.c_void_p),
        ("unclamp", C.c_void_p),
        ("inject_v", C.c_void_p),
        ("rec_s", C.c_void_p),
        ("rec_v", C.c_void_p),
        ("rec_count", C.c_void_p),
        ("_u", _CurrentOrNeuronParams),
    ]


class _SparseFields(C.Structure):
    _fields_ = [("sp_rowptr", C.c_void_p), ("sp_col", C.c_void_p), ("nnz", C.c_int32)]


class _Conv3dFields(C.Structure):
    _fields_ = [("din", C.c_int32), ("dout", C.c_int32), ("kd", C.c_int32), ("sd", C.c_int32), ("pd", C.c_int32),
                ("dd", C.c_int32)]


class _MeanFieldFields(C.Structure):
    _fields_ = [("mf_off", C.c_void_p), ("mf_stride", C.c_int32)]


class _WeightNormFields(C.Structure):
    _fields_ = [("norm_t", C.c_void_p), ("norm_step", C.c_int32)]


class _SparseOrConv3d(C.Union):
    """The storage SNN_CONN_SPARSE's pattern, the depth axis of SNN_CONN_CONV3D / SNN_CONN_LOCAL3D /
    SNN_CONN_MAXPOOL3D, SNN_CONN_MEANFIELD's offset map and the SNN_CONN_WNORM norm of a dense or MCC connection share
    (a connection is only one of these kinds)."""

    _anonymous_ = ("_sparse", "_conv3d", "_meanfield", "_wnorm")
    _fields_ = [("_sparse", _SparseFields), ("_conv3d", _Conv3dFields), ("_meanfield", _MeanFieldFields),
                ("_wnorm", _WeightNormFields)]


class _FeatureFields(C.Structure):
    _fields_ = [("f_prob", C.c_void_p), ("f_mask", C.c_void_p), ("f_int", C.c_void_p),
                ("draw_seed", C.c_uint32), ("draw_step", C.c_uint32), ("draw_conn", C.c_uint32)]


class _SynapseFields(C.Structure):
    _fields_ = [("wmin_t", C.c_void_p), ("wmax_t", C.c_void_p), ("nu0_t", C.c_void_p), ("nu1_t", C.c_void_p),
                ("wmin_form", C.c_int8), ("wmax_form", C.c_int8), ("nu0_form", C.c_int8), ("nu1_form", C.c_int8)]


class _FeaturesOrSynapse(C.Union):
    """The storage SNN_CONN_MCC's features and SNN_CONN_DENSE's per-synapse tensors share (a connection is never both)."""

    _anonymous_ = ("_feat", "_syn")
    _fields_ = [("_feat", _FeatureFields), ("_syn", _SynapseFields)]


class _RewardFields(C.Structure):
    _fields_ = [("reward", C.c_float), ("a_plus", C.c_float), ("a_minus", C.c_float), ("p_plus_decay", C.c_float),
                ("p_minus_decay", C.c_float), ("p_plus", C.c_void_p), ("p_minus", C.c_void_p), ("elig", C.c_void_p),
                ("mst_spre", C.c_void_p), ("mst_spost", C.c_void_p)]


class _AverageFields(C.Structure):
    _fields_ = [("avg_pre", C.c_void_p), ("avg_post", C.c_void_p), ("avg_rows", C.c_void_p), ("avg_cols", C.c_void_p),
                ("avg_k", C.c_int32), ("avg_idx_pre", C.c_int32), ("avg_idx_post", C.c_int32), ("avg_continues", C.c_int32)]


class _RewardOrAverage(C.Union):
    """The storage the reward-modulated rules' state and MCC PostPre's averaging state (SNN_RULE_AVG) share."""

    _anonymous_ = ("_reward", "_avg")
    _fields_ = [("_reward", _RewardFields), ("_avg", _AverageFields)]


class SnnConn(C.Structure):
    _anonymous_ = ("_r", "_u", "_f")
    _fields_ = [
        ("kind", C.c_int32),
        ("src", C.c_int32),
        ("tgt", C.c_int32),
        ("rule", C.c_int32),
        ("reduction", C.c_int32),
        ("has_norm", C.c_int32),
        ("norm_abs", C.c_int32),
        ("has_clamp", C.c_int32),
        ("structure", C.c_int32),
        ("nu0", C.c_float),
        ("nu1", C.c_float),
        ("wmin", C.c_float),
        ("wmax", C.c_float),
        ("weight_decay", C.c_float),
        ("dt_scale", C.c_float),
        ("norm", C.c_float),
        ("structure_val", C.c_float),
        ("w", C.c_void_p),
        ("b", C.c_void_p),
        ("cin", C.c_int32), ("hin", C.c_int32), ("win", C.c_int32),
        ("cout", C.c_int32), ("hout", C.c_int32), ("wout", C.c_int32),
        ("kh", C.c_int32), ("kw", C.c_int32), ("sh", C.c_int32), ("sw", C.c_int32),
        ("ph", C.c_int32), ("pw", C.c_int32), ("dh", C.c_int32), ("dw", C.c_int32),
        ("_r", _RewardOrAverage),
        ("mask", C.c_void_p),
        ("e_trace", C.c_void_p),
        ("e_trace_decay", C.c_float),
        ("tc_e_trace", C.c_float),
        ("et_coef", C.c_float),
        ("_u", _SparseOrConv3d),
        ("_f", _FeaturesOrSynapse),
        ("pool_rates", C.c_void_p),
        ("pool_decay", C.c_float),
    ]


class SnnNet(C.Structure):
    _fields_ = [
        ("abi_version", C.c_int32),
        ("n_layers", C.c_int32),
        ("n_conns", C.c_int32),
        ("learning", C.c_int32),
        ("layers", SnnLayer * SNN_MAX_LAYERS),
        ("conns", SnnConn * SNN_MAX_CONNS),
    ]


class SnnRunOpts(C.Structure):
    _fields_ = [
        ("T", C.c_int32),
        ("B", C.c_int32),
        ("normalize", C.c_int32),
        ("tier", C.c_int32),
        ("seed", C.c_uint32),
        ("step_offset", C.c_uint32),
        ("err_flag", C.c_void_p),
        ("one_step", C.c_int32),
        ("delta_w", C.c_void_p),
        ("delta_theta", C.c_void_p),
    ]


def _fmix32(h: int) -> int:
    h &= 0xFFFFFFFF
    h ^= h >> 16
    h = (h * 0x85EBCA6B) & 0xFFFFFFFF
    h ^= h >> 13
    h = (h * 0xC2B2AE35) & 0xFFFFFFFF
    h ^= h >> 16
    return h


def one_spike_hash(seed: int, t: int, layer: int, b: int, j: int) -> int:
    """Python restatement of ``snn_one_spike_hash`` (include/snn_b200.h)."""
    h = _fmix32((seed ^ (0x9E3779B9 * (t + 1))) & 0xFFFFFFFF)
    h = _fmix32((h + 0x85EBCA6B * (layer + 1) + b) & 0xFFFFFFFF)
    h = _fmix32((h ^ (0xC2B2AE35 * (j + 1))) & 0xFFFFFFFF)
    return h


def one_spike_key(seed: int, t: int, layer: int, b: int, j: int) -> int:
    return ((one_spike_hash(seed, t, layer, b, j) | 0x80000000) << 32) | j


def synapse_draw(seed: int, t: int, conn: int, i: int, j: int) -> int:
    """Python restatement of ``snn_synapse_draw`` (include/snn_b200.h): the Probability feature's hash of synapse (i, j)
    of connection ``conn`` at step ``t``."""
    h = _fmix32((seed ^ 0x53594E41) & 0xFFFFFFFF)
    h = _fmix32((h ^ (0x9E3779B9 * (t + 1))) & 0xFFFFFFFF)
    h = _fmix32((h ^ (0x85EBCA6B * (conn + 1))) & 0xFFFFFFFF)
    h = _fmix32((h ^ (0xC2B2AE35 * (i + 1))) & 0xFFFFFFFF)
    return _fmix32((h ^ (0x27D4EB2F * (j + 1))) & 0xFFFFFFFF)


def synapse_transmits(h: int, p: float) -> bool:
    """``snn_synapse_transmits``: (h >> 8) * 2**-24 < p, compared in float32 (exact: both sides are float32 values)."""
    import numpy as np

    return bool(np.float32((h >> 8) * 2.0**-24) < np.float32(p))
