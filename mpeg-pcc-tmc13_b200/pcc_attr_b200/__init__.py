"""ctypes binding of the C ABI in include/pcc_attr_b200.h (used by the tests
and bench.py; the product itself is the C ABI + CUDA kernels).

There is no CPU fallback: importing works anywhere, but every compute call
raises if libpcc_attr_b200.so is missing or no sm_90 (H100) device is present."""
import ctypes as C
import os

import numpy as np

# one hardware queue per library lane (see the header: the application sets it,
# before its CUDA context exists; this binding is the application here)
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(os.path.dirname(_HERE), "libpcc_attr_b200.so")

MAX_QP_LAYERS = 32
MAX_AC_QP_LAYERS = 32


class RahtParams(C.Structure):
    """pccb200_raht_params <- pcc::RahtPredictionParams (tmc3/hls.h:439-466)"""
    _fields_ = [
        ("prediction_enabled", C.c_int32),
        ("integer_haar", C.c_int32),
        ("prediction_threshold0", C.c_int32),
        ("prediction_threshold1", C.c_int32),
        ("subnode_prediction_enabled", C.c_int32),
        ("prediction_search_range", C.c_int32),
        ("pred_weight_parent", C.c_int32 * 19),
        ("pred_weight_child", C.c_int32 * 12),
        ("raht_extension", C.c_int32),
    ]


class QpSet(C.Structure):
    """pccb200_qpset <- pcc::QpSet (tmc3/quantization.h:123-137)"""
    _fields_ = [
        ("num_layers", C.c_int32),
        ("layers", (C.c_int32 * 2) * MAX_QP_LAYERS),
        ("max_qp", C.c_int32),
        ("fixed_point_qp_offset", C.c_int32),
        ("num_ac_coeff_qp_layers", C.c_int32),
        ("ac_coeff_qps", ((C.c_int32 * 2) * 7) * MAX_AC_QP_LAYERS),
    ]


class Predictor(C.Structure):
    _fields_ = [
        ("neighbor_count", C.c_uint32),
        ("predictor_index", C.c_uint32 * 3),
        ("weight", C.c_uint32 * 3),
    ]


MAX_LODS = 32
MAX_LIFT_SETS = 4


class LodParams(C.Structure):
    """pccb200_lod_params <- LoD fields of pcc::AttributeParameterSet (tmc3/hls.h:795-857)"""
    _fields_ = [
        ("num_detail_levels", C.c_int32),
        ("lod_decimation_type", C.c_int32),
        ("lod_sampling_period", C.c_int32 * MAX_LODS),
        ("dist2", C.c_int32),
        ("num_pred_nearest_neighbours", C.c_int32),
        ("inter_lod_search_range", C.c_int32),
        ("intra_lod_search_range", C.c_int32),
        ("intra_lod_prediction_skip_layers", C.c_int32),
        ("prediction_with_distribution", C.c_int32),
        ("lod_neigh_bias", C.c_int32 * 3),
        ("pred_weight_blending", C.c_int32),
    ]


class LodScalable(C.Structure):
    """pccb200_lod_scalable: scalable lifting beside a LodParams.  geom_num_points
    0 means n (the encoder, and every full decode)."""
    _fields_ = [
        ("max_neigh_range", C.c_int32),
        ("min_geom_node_size_log2", C.c_int32),
        ("geom_num_points", C.c_int64),
        ("reserved", C.c_int32),
    ]


# levels of detail of scalable lifting (maxNumDetailLevels)
SCALABLE_LODS = 21

PREDICTOR_DTYPE = np.dtype([("neighbor_count", "<u4"), ("predictor_index", "<u4", 3),
                            ("weight", "<u4", 3)])

EXPORTS = [
    "pccb200_abi_version", "pccb200_attr_lift_decode", "pccb200_attr_lift_decode_lod",
    "pccb200_attr_lift_decode_multi", "pccb200_attr_lift_decode_multi_batch",
    "pccb200_attr_lift_decode_multi_batch_dev", "pccb200_attr_lift_decode_multi_dev",
    "pccb200_attr_lift_decode_scalable", "pccb200_attr_lift_decode_scalable_dev",
    "pccb200_attr_lift_decode_slices", "pccb200_attr_lift_decode_slices_dev",
    "pccb200_attr_lift_encode", "pccb200_attr_lift_encode_lod",
    "pccb200_attr_lift_encode_multi", "pccb200_attr_lift_encode_multi_batch",
    "pccb200_attr_lift_encode_multi_batch_dev", "pccb200_attr_lift_encode_multi_dev",
    "pccb200_attr_lift_encode_scalable", "pccb200_attr_lift_encode_scalable_dev",
    "pccb200_attr_lift_encode_slices", "pccb200_attr_lift_encode_slices_dev",
    "pccb200_attr_pred_decode_lod", "pccb200_attr_pred_decode_multi_batch",
    "pccb200_attr_pred_decode_multi_batch_dev",
    "pccb200_attr_raht_decode",
    "pccb200_attr_raht_decode_multi", "pccb200_attr_raht_decode_multi_batch",
    "pccb200_attr_raht_decode_multi_batch_dev", "pccb200_attr_raht_decode_multi_dev",
    "pccb200_attr_raht_decode_slices_dev", "pccb200_attr_raht_encode",
    "pccb200_attr_raht_encode_multi", "pccb200_attr_raht_encode_multi_batch",
    "pccb200_attr_raht_encode_multi_batch_dev", "pccb200_attr_raht_encode_multi_dev",
    "pccb200_attr_raht_encode_slices", "pccb200_attr_raht_encode_slices_dev",
    "pccb200_attr_raht_encode_symbols", "pccb200_attr_spherical_positions",
    "pccb200_coeff_symbols", "pccb200_estimate_dist2", "pccb200_kernel_launch_count",
    "pccb200_last_error", "pccb200_lift_dequantize", "pccb200_lift_forward",
    "pccb200_lift_inverse", "pccb200_lift_quantize", "pccb200_lod_build",
    "pccb200_lod_build_scalable", "pccb200_lod_create",
    "pccb200_lod_destroy", "pccb200_lod_import", "pccb200_lod_info", "pccb200_lod_reusable", "pccb200_morton_sort",
    "pccb200_offset_and_scale", "pccb200_profile_enable", "pccb200_profile_read",
    "pccb200_profile_reset", "pccb200_quant_weights", "pccb200_quant_weights_fixed",
    "pccb200_quant_weights_scalable", "pccb200_raht_forward", "pccb200_raht_inverse",
    "pccb200_raht_params_default", "pccb200_raht_set_prediction_weights", "pccb200_recolour",
    "pccb200_recolour_exact", "pccb200_recolour_exact_multi_batch",
    "pccb200_recolour_exact_multi_batch_dev", "pccb200_recolour_multi", "pccb200_recolour_multi_batch", "pccb200_recolour_multi_batch_dev",
    "pccb200_recolour_multi_dev", "pccb200_recolour_params_default", "pccb200_set_device",
    "pccb200_time_begin", "pccb200_time_end", "pccb200_xyz_to_rpl",
]
NUM_PHASES = 8
PHASE_NAMES = ["sort", "tree_build", "block_transform", "tail", "gather_scatter", "lifting",
               "block_geometry", "block_schedule"]


class PccB200Error(RuntimeError):
    pass


_lib = None


def lib():
    """Load the CUDA library; raises loudly if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise PccB200Error(
                f"{LIB_PATH} not found: build it with `make -C mpeg-pcc-tmc13_b200` "
                "(or __graft_entry__.build()); there is no CPU fallback")
        l = C.CDLL(LIB_PATH)
        l.pccb200_last_error.restype = C.c_char_p
        l.pccb200_kernel_launch_count.restype = C.c_uint64
        _lib = l
    return _lib


def _check(rc):
    if rc != 0:
        raise PccB200Error(f"pccb200 status {rc}: {lib().pccb200_last_error().decode()}")


def _p(a, t):
    if a is None:
        return None
    if hasattr(a, "data_ptr"):  # torch CPU tensor (e.g. pinned)
        return C.cast(a.data_ptr(), C.POINTER(t))
    return a.ctypes.data_as(C.POINTER(t))


def default_params():
    p = RahtParams()
    lib().pccb200_raht_params_default(C.byref(p))
    return p


def kernel_launch_count():
    return int(lib().pccb200_kernel_launch_count())


def set_device(i):
    _check(lib().pccb200_set_device(C.c_int(i)))


def morton_sort(xyz):
    xyz = np.ascontiguousarray(xyz, dtype=np.int32)
    n = xyz.shape[0]
    keys = np.empty(n, dtype=np.int64)
    order = np.empty(n, dtype=np.int32)
    _check(lib().pccb200_morton_sort(_p(xyz, C.c_int32), C.c_int32(n), _p(keys, C.c_int64),
                                     _p(order, C.c_int32)))
    return keys, order


def raht_forward(params, qpset, morton, attrs, qpoffs=None):
    """-> (reconstructed attrs [N,A], coefficients [A,N])"""
    attrs = np.ascontiguousarray(attrs, dtype=np.int32).copy()
    n, a = attrs.shape
    morton = np.ascontiguousarray(morton, dtype=np.int64)
    coeffs = np.empty((a, n), dtype=np.int32)
    if qpoffs is not None:
        qpoffs = np.ascontiguousarray(qpoffs, dtype=np.int32)
    _check(lib().pccb200_raht_forward(C.byref(params), C.byref(qpset), _p(qpoffs, C.c_int32),
                                      _p(morton, C.c_int64), _p(attrs, C.c_int32),
                                      C.c_int32(a), C.c_int32(n), _p(coeffs, C.c_int32)))
    return attrs, coeffs


def raht_inverse(params, qpset, morton, coeffs, qpoffs=None):
    coeffs = np.ascontiguousarray(coeffs, dtype=np.int32)
    a, n = coeffs.shape
    morton = np.ascontiguousarray(morton, dtype=np.int64)
    attrs = np.empty((n, a), dtype=np.int32)
    if qpoffs is not None:
        qpoffs = np.ascontiguousarray(qpoffs, dtype=np.int32)
    _check(lib().pccb200_raht_inverse(C.byref(params), C.byref(qpset), _p(qpoffs, C.c_int32),
                                      _p(morton, C.c_int64), _p(attrs, C.c_int32),
                                      C.c_int32(a), C.c_int32(n), _p(coeffs, C.c_int32)))
    return attrs


def attr_raht_encode_into(params, qpset, xyz, attrs_inout, coeffs_out, bitdepth=8,
                          qpoffs=None, slice_offsets=None):
    """Zero-copy form used by bench.py: arrays may be numpy or (pinned) torch
    CPU tensors; attrs_inout [N,A] int32 is overwritten with the clipped
    reconstruction, coeffs_out [A,N] int32 receives the coefficients."""
    n, a = attrs_inout.shape
    if slice_offsets is None:
        _check(lib().pccb200_attr_raht_encode(
            C.byref(params), C.byref(qpset), _p(qpoffs, C.c_int32), _p(xyz, C.c_int32),
            _p(attrs_inout, C.c_int32), C.c_int32(a), C.c_int32(n), C.c_int32(bitdepth),
            _p(coeffs_out, C.c_int32)))
    else:
        so = np.ascontiguousarray(slice_offsets, dtype=np.int64)
        _check(lib().pccb200_attr_raht_encode_slices(
            C.byref(params), C.byref(qpset), _p(qpoffs, C.c_int32), _p(xyz, C.c_int32),
            _p(attrs_inout, C.c_int32), C.c_int32(a), C.c_int32(bitdepth),
            _p(so, C.c_int64), C.c_int32(len(so) - 1), _p(coeffs_out, C.c_int32)))


def attr_raht_encode(params, qpset, xyz, attrs, bitdepth=8, qpoffs=None, slice_offsets=None):
    xyz = np.ascontiguousarray(xyz, dtype=np.int32)
    attrs = np.ascontiguousarray(attrs, dtype=np.int32).copy()
    n, a = attrs.shape
    coeffs = np.empty((a, n), dtype=np.int32)
    if qpoffs is not None:
        qpoffs = np.ascontiguousarray(qpoffs, dtype=np.int32)
    attr_raht_encode_into(params, qpset, xyz, attrs, coeffs, bitdepth, qpoffs, slice_offsets)
    return attrs, coeffs


def attr_raht_decode(params, qpset, xyz, coeffs, bitdepth=8, qpoffs=None):
    xyz = np.ascontiguousarray(xyz, dtype=np.int32)
    coeffs = np.ascontiguousarray(coeffs, dtype=np.int32)
    a, n = coeffs.shape
    attrs = np.empty((n, a), dtype=np.int32)
    if qpoffs is not None:
        qpoffs = np.ascontiguousarray(qpoffs, dtype=np.int32)
    _check(lib().pccb200_attr_raht_decode(
        C.byref(params), C.byref(qpset), _p(qpoffs, C.c_int32), _p(xyz, C.c_int32),
        _p(attrs, C.c_int32), C.c_int32(a), C.c_int32(n), C.c_int32(bitdepth),
        _p(coeffs, C.c_int32)))
    return attrs


def _multi_args(qpsets, arrays_attrs, arrays_coef, bitdepths):
    k = len(qpsets)
    QP = C.POINTER(QpSet) * k
    IP = C.POINTER(C.c_int32) * k
    qp = QP(*[C.pointer(q) for q in qpsets])
    at = IP(*[_p(a, C.c_int32) for a in arrays_attrs])
    co = IP(*[_p(c, C.c_int32) for c in arrays_coef])
    na = (C.c_int32 * k)(*[int(a.shape[1]) for a in arrays_attrs])
    bd = (C.c_int32 * k)(*bitdepths)
    return qp, at, co, na, bd


def attr_raht_encode_multi_into(params, qpsets, xyz, attrs_inout, coeffs_out, bitdepths=None):
    """Several attributes of one slice in one pass (zero-copy form).
    attrs_inout[s]: [N, A_s] int32 (overwritten with the reconstruction),
    coeffs_out[s]: [A_s, N] int32."""
    k = len(qpsets)
    bitdepths = bitdepths or [8] * k
    n = attrs_inout[0].shape[0]
    qp, at, co, na, bd = _multi_args(qpsets, attrs_inout, coeffs_out, bitdepths)
    _check(lib().pccb200_attr_raht_encode_multi(
        C.byref(params), C.c_int32(k), qp, _p(xyz, C.c_int32), at, na, bd, C.c_int32(n), co))


def attr_raht_encode_multi(params, qpsets, xyz, attrs, bitdepths=None):
    xyz = np.ascontiguousarray(xyz, dtype=np.int32)
    a = [np.ascontiguousarray(x, dtype=np.int32).copy() for x in attrs]
    c = [np.empty((x.shape[1], x.shape[0]), dtype=np.int32) for x in a]
    attr_raht_encode_multi_into(params, qpsets, xyz, a, c, bitdepths)
    return a, c


def attr_raht_decode_multi(params, qpsets, xyz, coeffs, bitdepths=None):
    xyz = np.ascontiguousarray(xyz, dtype=np.int32)
    k = len(qpsets)
    bitdepths = bitdepths or [8] * k
    c = [np.ascontiguousarray(x, dtype=np.int32) for x in coeffs]
    a = [np.empty((x.shape[1], x.shape[0]), dtype=np.int32) for x in c]
    n = a[0].shape[0]
    qp, at, co, na, bd = _multi_args(qpsets, a, c, bitdepths)
    _check(lib().pccb200_attr_raht_decode_multi(
        C.byref(params), C.c_int32(k), qp, _p(xyz, C.c_int32), at, na, bd, C.c_int32(n), co))
    return a


def attr_raht_encode_multi_dev(params, qpsets, d_xyz, d_attrs, d_coefs, n, num_attrs, bitdepths=None):
    """device pointers (ints) for xyz, each attribute array and each coefficient array"""
    k = len(qpsets)
    bitdepths = bitdepths or [8] * k
    QP = C.POINTER(QpSet) * k
    VP = C.c_void_p * k
    qp = QP(*[C.pointer(q) for q in qpsets])
    at = VP(*d_attrs)
    co = VP(*d_coefs)
    na = (C.c_int32 * k)(*num_attrs)
    bd = (C.c_int32 * k)(*bitdepths)
    _check(lib().pccb200_attr_raht_encode_multi_dev(
        C.byref(params), C.c_int32(k), qp, C.c_void_p(d_xyz), at, na, bd, C.c_int32(n), co))


def _batch_args(qpsets, units_attrs, units_coefs, bitdepths):
    k = len(qpsets)
    m = len(units_attrs)
    QP = C.POINTER(QpSet) * k
    VP = C.c_void_p * (m * k)
    qp = QP(*[C.pointer(q) for q in qpsets])

    def ptr(x):
        return x if isinstance(x, int) else x.data_ptr() if hasattr(x, "data_ptr") else x.ctypes.data

    at = VP(*[ptr(a) for u in units_attrs for a in u])
    co = VP(*[ptr(c) for u in units_coefs for c in u])
    bd = (C.c_int32 * k)(*bitdepths)
    return qp, at, co, bd


def attr_raht_encode_multi_batch_into(params, qpsets, xyzs, attrs_inout, coeffs_out, bitdepths=None):
    """Many coding units (slices / frames) in one call, zero-copy form.
    xyzs[u]: [N_u, 3] int32; attrs_inout[u][s]: [N_u, A_s] int32 (overwritten
    with the reconstruction); coeffs_out[u][s]: [A_s, N_u] int32."""
    k = len(qpsets)
    m = len(xyzs)
    bitdepths = bitdepths or [8] * k
    qp, at, co, bd = _batch_args(qpsets, attrs_inout, coeffs_out, bitdepths)
    na = (C.c_int32 * k)(*[int(a.shape[1]) for a in attrs_inout[0]])
    xp = (C.c_void_p * m)(*[x.data_ptr() if hasattr(x, "data_ptr") else x.ctypes.data for x in xyzs])
    ns = (C.c_int32 * m)(*[int(x.shape[0]) for x in xyzs])
    _check(lib().pccb200_attr_raht_encode_multi_batch(
        C.byref(params), C.c_int32(k), qp, C.c_int32(m), xp, at, na, bd, ns, co))


def attr_raht_encode_multi_batch(params, qpsets, xyzs, attrs, bitdepths=None):
    """-> (recs[u][s], coefs[u][s])"""
    xyzs = [np.ascontiguousarray(x, dtype=np.int32) for x in xyzs]
    a = [[np.ascontiguousarray(x, dtype=np.int32).copy() for x in u] for u in attrs]
    c = [[np.empty((x.shape[1], x.shape[0]), dtype=np.int32) for x in u] for u in a]
    attr_raht_encode_multi_batch_into(params, qpsets, xyzs, a, c, bitdepths)
    return a, c


def attr_raht_decode_multi_batch(params, qpsets, xyzs, coeffs, bitdepths=None):
    """-> recs[u][s]"""
    k = len(qpsets)
    m = len(xyzs)
    bitdepths = bitdepths or [8] * k
    xyzs = [np.ascontiguousarray(x, dtype=np.int32) for x in xyzs]
    c = [[np.ascontiguousarray(x, dtype=np.int32) for x in u] for u in coeffs]
    a = [[np.empty((x.shape[1], x.shape[0]), dtype=np.int32) for x in u] for u in c]
    qp, at, co, bd = _batch_args(qpsets, a, c, bitdepths)
    na = (C.c_int32 * k)(*[int(x.shape[1]) for x in a[0]])
    xp = (C.c_void_p * m)(*[x.ctypes.data for x in xyzs])
    ns = (C.c_int32 * m)(*[int(x.shape[0]) for x in xyzs])
    _check(lib().pccb200_attr_raht_decode_multi_batch(
        C.byref(params), C.c_int32(k), qp, C.c_int32(m), xp, at, na, bd, ns, co))
    return a


def attr_raht_multi_batch_dev(forward, params, qpsets, d_xyzs, d_attrs, d_coefs, ns, num_attrs,
                              bitdepths=None):
    """device pointers (ints): d_xyzs[u], d_attrs[u][s], d_coefs[u][s]; ns[u] points"""
    k = len(qpsets)
    m = len(d_xyzs)
    bitdepths = bitdepths or [8] * k
    qp, at, co, bd = _batch_args(qpsets, d_attrs, d_coefs, bitdepths)
    na = (C.c_int32 * k)(*num_attrs)
    xp = (C.c_void_p * m)(*d_xyzs)
    nn = (C.c_int32 * m)(*ns)
    fn = (lib().pccb200_attr_raht_encode_multi_batch_dev if forward
          else lib().pccb200_attr_raht_decode_multi_batch_dev)
    _check(fn(C.byref(params), C.c_int32(k), qp, C.c_int32(m), xp, at, na, bd, nn, co))


class RecolourParams(C.Structure):
    _fields_ = [("dist_offset_fwd", C.c_double), ("dist_offset_bwd", C.c_double),
                ("max_geometry_dist2_fwd", C.c_double), ("max_geometry_dist2_bwd", C.c_double),
                ("max_attribute_dist2_fwd", C.c_double), ("max_attribute_dist2_bwd", C.c_double),
                ("search_range", C.c_int32), ("num_neighbours_fwd", C.c_int32),
                ("num_neighbours_bwd", C.c_int32), ("use_dist_weighted_avg_fwd", C.c_int32),
                ("use_dist_weighted_avg_bwd", C.c_int32),
                ("skip_avg_if_identical_source_point_present_fwd", C.c_int32),
                ("skip_avg_if_identical_source_point_present_bwd", C.c_int32),
                ("reserved", C.c_int32)]


def default_recolour_params():
    p = RecolourParams()
    lib().pccb200_recolour_params_default(C.byref(p))
    return p


def recolour(params, source_xyz, source_attrs, target_xyz, scale=1.0, offset=(0, 0, 0), bitdepth=8):
    """attribute transfer source -> target (pccb200_recolour); -> [n_target, A] int32"""
    sx = np.ascontiguousarray(source_xyz, dtype=np.int32)
    sa = np.ascontiguousarray(source_attrs, dtype=np.int32)
    tx = np.ascontiguousarray(target_xyz, dtype=np.int32)
    if sa.ndim == 1:
        sa = sa[:, None]
    a = sa.shape[1]
    out = np.zeros((tx.shape[0], a), dtype=np.int32)
    off = (C.c_int32 * 3)(*[int(v) for v in offset])
    _check(lib().pccb200_recolour(C.byref(params), _p(sx, C.c_int32), _p(sa, C.c_int32), C.c_int32(a),
                                  C.c_int32(sx.shape[0]), C.c_double(scale), off, _p(tx, C.c_int32),
                                  C.c_int32(tx.shape[0]), C.c_int32(bitdepth), _p(out, C.c_int32)))
    return out


def recolour_exact(params, source_xyz, source_attrs, target_xyz, scale=1.0, offset=(0, 0, 0),
                   bitdepth=8):
    """as recolour, with the reference's own neighbour search and list order
    (pccb200_recolour_exact): equal to recolourColour / recolourReflectance bit
    for bit; coordinates and offsets of |x| < 2^30; -> [n_target, A] int32"""
    sx = np.ascontiguousarray(source_xyz, dtype=np.int32)
    sa = np.ascontiguousarray(source_attrs, dtype=np.int32)
    tx = np.ascontiguousarray(target_xyz, dtype=np.int32)
    if sa.ndim == 1:
        sa = sa[:, None]
    a = sa.shape[1]
    out = np.zeros((tx.shape[0], a), dtype=np.int32)
    off = (C.c_int32 * 3)(*[int(v) for v in offset])
    _check(lib().pccb200_recolour_exact(C.byref(params), _p(sx, C.c_int32), _p(sa, C.c_int32), C.c_int32(a),
                                        C.c_int32(sx.shape[0]), C.c_double(scale), off, _p(tx, C.c_int32),
                                        C.c_int32(tx.shape[0]), C.c_int32(bitdepth), _p(out, C.c_int32)))
    return out


def _recolour_batch_args(sources, source_attrs, targets, scales, offsets, outs, bitdepths, ptr):
    """C arrays of a pccb200_recolour_multi_batch(_dev) call; source_attrs[u][s], outs[u][s]"""
    m, k = len(sources), len(source_attrs[0])
    VP = C.c_void_p * m
    AP = C.c_void_p * (m * k)
    return (C.c_int32(k), C.c_int32(m), VP(*[ptr(x) for x in sources]),
            (C.c_int32 * m)(*[int(x.shape[0]) for x in sources]),
            AP(*[ptr(a) for u in source_attrs for a in u]),
            (C.c_int32 * k)(*[int(a.shape[1]) for a in source_attrs[0]]),
            (C.c_int32 * k)(*bitdepths), (C.c_double * m)(*[float(s) for s in scales]),
            (C.c_int32 * (3 * m))(*[int(v) for o in offsets for v in o]),
            VP(*[ptr(x) for x in targets]), (C.c_int32 * m)(*[int(x.shape[0]) for x in targets]),
            AP(*[ptr(o) for u in outs for o in u]))


def recolour_multi(params, source_xyz, source_attrs, target_xyz, scale=1.0, offset=(0, 0, 0),
                   bitdepths=None):
    """several attribute sets on the same positions in one call
    (pccb200_recolour_multi); source_attrs[s]: [n_source, A_s] -> [[n_target, A_s] int32]"""
    sx = np.ascontiguousarray(source_xyz, dtype=np.int32)
    tx = np.ascontiguousarray(target_xyz, dtype=np.int32)
    sa = [np.ascontiguousarray(a, dtype=np.int32).reshape(sx.shape[0], -1) for a in source_attrs]
    k = len(sa)
    outs = [np.zeros((tx.shape[0], a.shape[1]), dtype=np.int32) for a in sa]
    IP = C.POINTER(C.c_int32) * k
    _check(lib().pccb200_recolour_multi(
        C.byref(params), C.c_int32(k), _p(sx, C.c_int32), C.c_int32(sx.shape[0]),
        IP(*[_p(a, C.c_int32) for a in sa]), (C.c_int32 * k)(*[a.shape[1] for a in sa]),
        (C.c_int32 * k)(*(bitdepths or [8] * k)), C.c_double(scale),
        (C.c_int32 * 3)(*[int(v) for v in offset]), _p(tx, C.c_int32), C.c_int32(tx.shape[0]),
        IP(*[_p(o, C.c_int32) for o in outs])))
    return outs


def recolour_multi_batch(params, sources, source_attrs, targets, scales, offsets, bitdepths=None,
                         exact=False):
    """many units (slices / frames) in one call (pccb200_recolour_multi_batch):
    sources[u] [n_source_u, 3], source_attrs[u][s] [n_source_u, A_s], targets[u],
    scales[u], offsets[u] (3) -> outs[u][s] [n_target_u, A_s] int32.  exact: the
    reference-exact path (pccb200_recolour_exact_multi_batch)"""
    sources = [np.ascontiguousarray(x, dtype=np.int32) for x in sources]
    targets = [np.ascontiguousarray(x, dtype=np.int32) for x in targets]
    sa = [[np.ascontiguousarray(a, dtype=np.int32).reshape(x.shape[0], -1) for a in u]
          for x, u in zip(sources, source_attrs)]
    outs = [[np.zeros((t.shape[0], a.shape[1]), dtype=np.int32) for a in u] for t, u in zip(targets, sa)]
    k = len(sa[0])
    args = _recolour_batch_args(sources, sa, targets, scales, offsets, outs, bitdepths or [8] * k,
                                lambda x: x.ctypes.data)
    fn = lib().pccb200_recolour_exact_multi_batch if exact else lib().pccb200_recolour_multi_batch
    _check(fn(C.byref(params), *args))
    return outs


def recolour_exact_multi_batch(params, sources, source_attrs, targets, scales, offsets, bitdepths=None):
    """recolour_multi_batch on the reference-exact path (pccb200_recolour_exact_multi_batch)"""
    return recolour_multi_batch(params, sources, source_attrs, targets, scales, offsets, bitdepths, exact=True)


def recolour_multi_batch_dev(params, sources, source_attrs, targets, scales, offsets, outs,
                             bitdepths=None, exact=False):
    """as recolour_multi_batch with contiguous int32 torch CUDA tensors (device
    pointers); the results are written into outs[u][s] [n_target_u, A_s].  The
    producing stream must be synchronised before the call (see the header).
    exact: the reference-exact path (pccb200_recolour_exact_multi_batch_dev)"""
    tensors = list(sources) + list(targets) + [a for u in source_attrs for a in u] + [o for u in outs for o in u]
    for t in tensors:
        if not (t.is_cuda and t.is_contiguous() and str(t.dtype) == "torch.int32"):
            raise PccB200Error("recolour_multi_batch_dev takes contiguous int32 CUDA tensors")
    k = len(source_attrs[0])
    args = _recolour_batch_args(sources, source_attrs, targets, scales, offsets, outs,
                                bitdepths or [8] * k, lambda x: x.data_ptr())
    fn = lib().pccb200_recolour_exact_multi_batch_dev if exact else lib().pccb200_recolour_multi_batch_dev
    _check(fn(C.byref(params), *args))


def recolour_exact_multi_batch_dev(params, sources, source_attrs, targets, scales, offsets, outs,
                                   bitdepths=None):
    """recolour_multi_batch_dev on the reference-exact path
    (pccb200_recolour_exact_multi_batch_dev)"""
    recolour_multi_batch_dev(params, sources, source_attrs, targets, scales, offsets, outs, bitdepths,
                             exact=True)


def quant_weights(preds, num_points_in_lod):
    preds = np.ascontiguousarray(preds, dtype=PREDICTOR_DTYPE)
    npl = np.ascontiguousarray(num_points_in_lod, dtype=np.uint32)
    n = preds.shape[0]
    qw = np.empty(n, dtype=np.uint64)
    _check(lib().pccb200_quant_weights(C.cast(preds.ctypes.data, C.POINTER(Predictor)),
                                       C.c_int32(n), _p(npl, C.c_uint32), C.c_int32(len(npl)),
                                       _p(qw, C.c_uint64)))
    return qw


def lift(forward, preds, qw, num_points_in_lod, attrs):
    preds = np.ascontiguousarray(preds, dtype=PREDICTOR_DTYPE)
    npl = np.ascontiguousarray(num_points_in_lod, dtype=np.uint32)
    qw = np.ascontiguousarray(qw, dtype=np.uint64)
    attrs = np.ascontiguousarray(attrs, dtype=np.int64).copy()
    if attrs.ndim == 1:
        attrs = attrs[:, None]
    n, a = attrs.shape
    fn = lib().pccb200_lift_forward if forward else lib().pccb200_lift_inverse
    _check(fn(C.cast(preds.ctypes.data, C.POINTER(Predictor)), _p(qw, C.c_uint64), C.c_int32(n),
              _p(npl, C.c_uint32), C.c_int32(len(npl)), _p(attrs, C.c_int64), C.c_int32(a)))
    return attrs


# ---- device-resident entry points (pointers are raw device addresses) ------

def time_begin():
    """Start of a device-timed region spanning every lane (CUDA events)."""
    _check(lib().pccb200_time_begin())


def time_end():
    """-> elapsed device milliseconds since time_begin()."""
    ms = C.c_double(0)
    _check(lib().pccb200_time_end(C.byref(ms)))
    return float(ms.value)


def attr_raht_encode_dev(params, qpset, d_xyz, d_attrs_inout, d_coeffs, n, a, bitdepth=8,
                         d_qpoffs=0, slice_offsets=None):
    so = np.ascontiguousarray(slice_offsets if slice_offsets is not None else [0, n],
                              dtype=np.int64)
    _check(lib().pccb200_attr_raht_encode_slices_dev(
        C.byref(params), C.byref(qpset), C.c_void_p(d_qpoffs or None), C.c_void_p(d_xyz),
        C.c_void_p(d_attrs_inout), C.c_int32(a), C.c_int32(bitdepth), _p(so, C.c_int64),
        C.c_int32(len(so) - 1), C.c_void_p(d_coeffs)))


def attr_raht_decode_dev(params, qpset, d_xyz, d_attrs_out, d_coeffs, n, a, bitdepth=8,
                         d_qpoffs=0, slice_offsets=None):
    so = np.ascontiguousarray(slice_offsets if slice_offsets is not None else [0, n],
                              dtype=np.int64)
    _check(lib().pccb200_attr_raht_decode_slices_dev(
        C.byref(params), C.byref(qpset), C.c_void_p(d_qpoffs or None), C.c_void_p(d_xyz),
        C.c_void_p(d_attrs_out), C.c_int32(a), C.c_int32(bitdepth), _p(so, C.c_int64),
        C.c_int32(len(so) - 1), C.c_void_p(d_coeffs)))


def profile_enable(on):
    lib().pccb200_profile_enable(C.c_int(1 if on else 0))


def profile_reset():
    lib().pccb200_profile_reset()


def profile_read():
    ms = (C.c_double * NUM_PHASES)()
    ln = (C.c_uint64 * NUM_PHASES)()
    lib().pccb200_profile_read(ms, ln)
    return {PHASE_NAMES[i]: (float(ms[i]), int(ln[i])) for i in range(NUM_PHASES)}


def lod_build(params, xyz):
    """-> (predictors[N] (PREDICTOR_DTYPE), indexes[N], num_points_in_lod[lods])"""
    xyz = np.ascontiguousarray(xyz, dtype=np.int32)
    n = xyz.shape[0]
    preds = np.zeros(n, dtype=PREDICTOR_DTYPE)
    indexes = np.zeros(n, dtype=np.uint32)
    npl = np.zeros(MAX_LODS, dtype=np.uint32)
    cnt = C.c_int32(0)
    _check(lib().pccb200_lod_build(C.byref(params), _p(xyz, C.c_int32), C.c_int32(n),
                                   C.cast(preds.ctypes.data, C.POINTER(Predictor)),
                                   _p(indexes, C.c_uint32), _p(npl, C.c_uint32), C.byref(cnt)))
    return preds, indexes, npl[:cnt.value].copy()


def lod_build_scalable(params, scal, xyz):
    """scalable lifting (pccb200_lod_build_scalable): params LodParams, scal
    LodScalable -> (predictors[N], indexes[N], num_points_in_lod[lods])"""
    xyz = np.ascontiguousarray(xyz, dtype=np.int32)
    n = xyz.shape[0]
    preds = np.zeros(n, dtype=PREDICTOR_DTYPE)
    indexes = np.zeros(n, dtype=np.uint32)
    npl = np.zeros(MAX_LODS, dtype=np.uint32)
    cnt = C.c_int32(0)
    _check(lib().pccb200_lod_build_scalable(
        C.byref(params), C.byref(scal), _p(xyz, C.c_int32), C.c_int32(n),
        C.cast(preds.ctypes.data, C.POINTER(Predictor)), _p(indexes, C.c_uint32),
        _p(npl, C.c_uint32), C.byref(cnt)))
    return preds, indexes, npl[:cnt.value].copy()


def lod_import(preds, indexes, num_points_in_lod, num_detail_levels, scal=None):
    """pccb200_lod_import: a level-of-detail handle over levels of detail the
    caller holds (preds: PREDICTOR_DTYPE [N], indexes [N], cumulative counts;
    scal: LodScalable for scalable lifting, or None) -> handle (an int);
    release it with lod_destroy"""
    preds = np.ascontiguousarray(preds, dtype=PREDICTOR_DTYPE)
    indexes = np.ascontiguousarray(indexes, dtype=np.uint32)
    npl = np.ascontiguousarray(num_points_in_lod, dtype=np.uint32)
    h = C.c_void_p()
    _check(lib().pccb200_lod_import(
        C.cast(preds.ctypes.data, C.POINTER(Predictor)), _p(indexes, C.c_uint32),
        C.c_int32(len(preds)), _p(npl, C.c_uint32), C.c_int32(len(npl)),
        C.c_int32(num_detail_levels), C.byref(scal) if scal is not None else None, C.byref(h)))
    return h.value


def lod_destroy(handle):
    lib().pccb200_lod_destroy(C.c_void_p(handle))


def attr_lift_encode_lod(handle, qpset, attrs, lcp_enabled=0, bitdepth=8, qpoffs=None):
    """pccb200_attr_lift_encode_lod -> (values [N,A] coding order, reconstruction
    [N,A] point order, lcp row of MAX_LODS entries)"""
    attrs = np.ascontiguousarray(attrs, dtype=np.int32).copy()
    n, a = attrs.shape
    values = np.zeros((n, a), dtype=np.int32)
    lcp = np.zeros(MAX_LODS, dtype=np.int8)
    if qpoffs is not None:
        qpoffs = np.ascontiguousarray(qpoffs, dtype=np.int32)
    _check(lib().pccb200_attr_lift_encode_lod(
        C.c_void_p(handle), C.byref(qpset), C.c_int32(lcp_enabled), _p(qpoffs, C.c_int32),
        _p(attrs, C.c_int32), C.c_int32(a), C.c_int32(bitdepth), _p(values, C.c_int32),
        _p(lcp, C.c_int8)))
    return values, attrs, lcp


def attr_lift_decode_lod(handle, qpset, values, lcp=None, bitdepth=8, qpoffs=None):
    """pccb200_attr_lift_decode_lod -> reconstruction [N,A] point order"""
    values = np.ascontiguousarray(values, dtype=np.int32)
    n, a = values.shape
    attrs = np.zeros((n, a), dtype=np.int32)
    l2 = None
    if lcp is not None:
        l2 = np.zeros(MAX_LODS, dtype=np.int8)
        l2[:len(lcp)] = lcp
    if qpoffs is not None:
        qpoffs = np.ascontiguousarray(qpoffs, dtype=np.int32)
    _check(lib().pccb200_attr_lift_decode_lod(
        C.c_void_p(handle), C.byref(qpset), C.c_int32(1 if lcp is not None else 0),
        _p(qpoffs, C.c_int32), _p(attrs, C.c_int32), C.c_int32(a), C.c_int32(bitdepth),
        _p(values, C.c_int32), _p(l2, C.c_int8)))
    return attrs


class PredParams(C.Structure):
    """pccb200_pred_params: the predicting transform's APS fields of one set"""
    _fields_ = [("max_num_direct_predictors", C.c_int32),
                ("direct_avg_predictor_disabled", C.c_int32),
                ("adaptive_prediction_threshold", C.c_int32),
                ("icp_enabled", C.c_int32)]


def _icp_row(icp):
    """None, or a host int8 row of MAX_LODS x 3 ICP coefficients"""
    if icp is None:
        return None
    row = np.zeros((MAX_LODS, 3), dtype=np.int8)
    icp = np.asarray(icp, dtype=np.int8).reshape(-1, 3)
    row[:len(icp)] = icp
    return row


def attr_pred_decode_lod(handle, qpset, pred, quant_neigh_weight, values, bitdepth=8,
                         qpoffs=None, icp=None):
    """pccb200_attr_pred_decode_lod: values [N, A] in coding order (as the
    reference's loop decodes them), icp [lods, 3] or None -> decoded
    attributes [N, A] in point order"""
    values = np.ascontiguousarray(values, dtype=np.int32)
    n, a = values.shape
    out = np.zeros((n, a), dtype=np.int32)
    if qpoffs is not None:
        qpoffs = np.ascontiguousarray(qpoffs, dtype=np.int32)
    qnw = (C.c_int32 * 3)(*[int(w) for w in quant_neigh_weight])
    row = _icp_row(icp)
    _check(lib().pccb200_attr_pred_decode_lod(
        C.c_void_p(handle), C.byref(qpset), C.byref(pred), qnw, _p(qpoffs, C.c_int32),
        _p(row, C.c_int8), _p(values, C.c_int32), C.c_int32(a), C.c_int32(bitdepth),
        _p(out, C.c_int32)))
    return out


def _pred_multi_args(lods, qnws, qpsets, preds, comps, bitdepths, xyzs, ns, qpos, values, icps,
                     outs):
    m, k = len(lods), len(qpsets)
    VP = C.c_void_p * (m * k)
    rows = [_icp_row(r) for u in icps for r in u] if icps is not None else None
    args = (C.c_int32(m), (C.POINTER(LodParams) * m)(*[C.pointer(lp) for lp in lods]),
            (C.c_int32 * (3 * m))(*[int(w) for q in qnws for w in q]), C.c_int32(k),
            (C.POINTER(QpSet) * k)(*[C.pointer(q) for q in qpsets]), (PredParams * k)(*preds),
            (C.c_int32 * k)(*comps), (C.c_int32 * k)(*(bitdepths or [8] * k)),
            (C.c_void_p * m)(*xyzs), (C.c_int32 * m)(*ns),
            (C.c_void_p * m)(*qpos) if qpos is not None else None, VP(*values),
            VP(*[None if r is None else r.ctypes.data for r in rows]) if rows is not None else None,
            VP(*outs))
    return args, rows


def attr_pred_decode_multi_batch(lods, quant_neigh_weights, qpsets, preds, xyzs, values,
                                 bitdepths=None, qpoffs=None, icps=None):
    """pccb200_attr_pred_decode_multi_batch: lods[u], quant_neigh_weights[u]
    (3 ints), xyzs[u] [N_u, 3], qpoffs[u] [N_u, 2] or None per unit; qpsets,
    preds (PredParams), bitdepths per set; values[u][s] [N_u, A_s] coding order,
    icps[u][s] [lods, 3] or None -> decoded attributes[u][s] in point order"""
    xyzs = [np.ascontiguousarray(x, dtype=np.int32) for x in xyzs]
    values = [[np.ascontiguousarray(v, dtype=np.int32).reshape(x.shape[0], -1) for v in u]
              for x, u in zip(xyzs, values)]
    outs = [[np.zeros_like(v) for v in u] for u in values]
    qpo = None
    if qpoffs is not None:
        qpo = [None if q is None else np.ascontiguousarray(q, dtype=np.int32) for q in qpoffs]
    args, _keep = _pred_multi_args(
        lods, quant_neigh_weights, qpsets, preds, [v.shape[1] for v in values[0]], bitdepths,
        [x.ctypes.data for x in xyzs], [x.shape[0] for x in xyzs],
        None if qpo is None else [None if q is None else q.ctypes.data for q in qpo],
        [v.ctypes.data for u in values for v in u], icps, [o.ctypes.data for u in outs for o in u])
    _check(lib().pccb200_attr_pred_decode_multi_batch(*args))
    return outs


def attr_pred_decode_multi_batch_dev(lods, quant_neigh_weights, qpsets, preds, comps, d_xyzs, ns,
                                     d_values, d_outs, bitdepths=None, d_qpoffs=None, icps=None):
    """pccb200_attr_pred_decode_multi_batch_dev: device pointers (ints) d_xyzs[u],
    d_qpoffs[u] (or None), d_values[u][s], d_outs[u][s]; comps[s] components
    per set, ns[u] points per unit; everything else as attr_pred_decode_multi_batch"""
    args, _keep = _pred_multi_args(
        lods, quant_neigh_weights, qpsets, preds, comps, bitdepths, list(d_xyzs), list(ns),
        list(d_qpoffs) if d_qpoffs is not None else None, [v for u in d_values for v in u],
        icps, [o for u in d_outs for o in u])
    _check(lib().pccb200_attr_pred_decode_multi_batch_dev(*args))


def attr_lift_encode(lod_params, qpset, xyz, attrs, lcp_enabled=0, bitdepth=8, qpoffs=None):
    """-> (values [N,A] coding order, reconstruction [N,A] point order, lcp coefficients)"""
    xyz = np.ascontiguousarray(xyz, dtype=np.int32)
    attrs = np.ascontiguousarray(attrs, dtype=np.int32).copy()
    n, a = attrs.shape
    values = np.zeros((n, a), dtype=np.int32)
    lcp = np.zeros(MAX_LODS, dtype=np.int8)
    if qpoffs is not None:
        qpoffs = np.ascontiguousarray(qpoffs, dtype=np.int32)
    _check(lib().pccb200_attr_lift_encode(
        C.byref(lod_params), C.byref(qpset), C.c_int32(lcp_enabled), _p(qpoffs, C.c_int32),
        _p(xyz, C.c_int32), _p(attrs, C.c_int32), C.c_int32(a), C.c_int32(n), C.c_int32(bitdepth),
        _p(values, C.c_int32), _p(lcp, C.c_int8)))
    return values, attrs, lcp[:lod_params.num_detail_levels].copy()


def attr_lift_slices_dev(forward, lod_params, qpset, lcp_enabled, d_xyz, d_attrs, a, slice_offsets,
                         d_values, lcp, bitdepth=8, d_qpoffs=None):
    """device pointers (ints) for xyz / attrs (coded in place) / values; slice_offsets
    (host, int64, numSlices + 1); lcp: host int8 [numSlices, MAX_LODS] (out when forward)"""
    so = np.ascontiguousarray(slice_offsets, dtype=np.int64)
    ns = len(so) - 1
    fn = (lib().pccb200_attr_lift_encode_slices_dev if forward
          else lib().pccb200_attr_lift_decode_slices_dev)
    _check(fn(C.byref(lod_params), C.byref(qpset), C.c_int32(lcp_enabled),
              C.c_void_p(d_qpoffs) if d_qpoffs else None, C.c_void_p(d_xyz), C.c_void_p(d_attrs),
              C.c_int32(a), C.c_int32(bitdepth), _p(so, C.c_int64), C.c_int32(ns),
              C.c_void_p(d_values), _p(lcp, C.c_int8)))


def attr_lift_decode(lod_params, qpset, xyz, values, lcp=None, bitdepth=8, qpoffs=None):
    xyz = np.ascontiguousarray(xyz, dtype=np.int32)
    values = np.ascontiguousarray(values, dtype=np.int32)
    n, a = values.shape
    attrs = np.zeros((n, a), dtype=np.int32)
    l2 = None
    if lcp is not None:
        l2 = np.zeros(MAX_LODS, dtype=np.int8)
        l2[:len(lcp)] = lcp
    _check(lib().pccb200_attr_lift_decode(
        C.byref(lod_params), C.byref(qpset), C.c_int32(1 if lcp is not None else 0),
        _p(qpoffs, C.c_int32), _p(xyz, C.c_int32), _p(attrs, C.c_int32), C.c_int32(a), C.c_int32(n),
        C.c_int32(bitdepth), _p(values, C.c_int32), _p(l2, C.c_int8)))
    return attrs


def _lift_multi_args(lods, qpsets, lcp_enabled, xyzs, attrs, values, lcps, bitdepths, ptr):
    """C arguments of a pccb200_attr_lift_*_multi_batch(_dev) call: attrs[u][s],
    values[u][s] (anything ptr() maps to an address), lcps[u][s] host int8 rows
    of MAX_LODS entries or None"""
    m, k = len(xyzs), len(qpsets)
    VP = C.c_void_p * (m * k)
    return (C.c_int32(m), (C.POINTER(LodParams) * m)(*[C.pointer(lp) for lp in lods]), C.c_int32(k),
            (C.POINTER(QpSet) * k)(*[C.pointer(q) for q in qpsets]),
            (C.c_int32 * k)(*[int(e) for e in (lcp_enabled or [0] * k)]),
            (C.c_void_p * m)(*[ptr(x) for x in xyzs]),
            (C.c_int32 * m)(*[int(x.shape[0]) for x in xyzs]),
            VP(*[ptr(a) for u in attrs for a in u]),
            (C.c_int32 * k)(*[int(a.shape[1]) for a in attrs[0]]),
            (C.c_int32 * k)(*(bitdepths or [8] * k)),
            VP(*[ptr(v) for u in values for v in u]),
            VP(*[None if r is None else r.ctypes.data for u in lcps for r in u]))


def attr_lift_multi_batch(forward, lods, qpsets, xyzs, data, lcp_enabled=None, bitdepths=None,
                          lcps=None):
    """Several attribute sets of many units (slices / frames) in one lifting call
    (pccb200_attr_lift_{en,de}code_multi_batch).  lods[u]: LodParams of unit u,
    xyzs[u]: [N_u, 3]; qpsets, lcp_enabled, bitdepths: per set.
    forward: data[u][s] = attributes [N_u, A_s] -> (values[u][s] coding order,
    reconstruction[u][s], lcp[u][s] (num_detail_levels of lods[u] entries)).
    Otherwise: data[u][s] = values, lcps[u][s] the encoder's lcp rows (or None)
    -> reconstruction[u][s]."""
    xyzs = [np.ascontiguousarray(x, dtype=np.int32) for x in xyzs]
    data = [[np.ascontiguousarray(a, dtype=np.int32).reshape(x.shape[0], -1) for a in u]
            for x, u in zip(xyzs, data)]
    if forward:
        attrs = [[a.copy() for a in u] for u in data]
        values = [[np.zeros_like(a) for a in u] for u in data]
        rows = [[np.zeros(MAX_LODS, dtype=np.int8) for _ in u] for u in data]
    else:
        attrs = [[np.zeros_like(a) for a in u] for u in data]
        values = data
        # a row that is not given stays null, so the library refuses a set that needs it
        rows = [[None] * len(u) for u in data]
        for u, lu in zip(rows, lcps if lcps is not None else []):
            for s, l in enumerate(lu if lu is not None else []):
                if l is not None:
                    u[s] = np.zeros(MAX_LODS, dtype=np.int8)
                    u[s][:len(l)] = l
    args = _lift_multi_args(lods, qpsets, lcp_enabled, xyzs, attrs, values, rows, bitdepths,
                            lambda x: x.ctypes.data)
    fn = (lib().pccb200_attr_lift_encode_multi_batch if forward
          else lib().pccb200_attr_lift_decode_multi_batch)
    _check(fn(*args))
    if not forward:
        return attrs
    return values, attrs, [[r[:lp.num_detail_levels].copy() for r in u] for lp, u in zip(lods, rows)]


def attr_lift_multi_encode(lod_params, qpsets, xyz, attrs, lcp_enabled=None, bitdepths=None):
    """several attribute sets of one slice in one lifting pass
    (pccb200_attr_lift_encode_multi): attrs[s] [N, A_s] -> (values[s] coding
    order, reconstruction[s], lcp[s] (num_detail_levels entries))"""
    xyz = np.ascontiguousarray(xyz, dtype=np.int32)
    attrs = [np.ascontiguousarray(a, dtype=np.int32).reshape(xyz.shape[0], -1).copy() for a in attrs]
    k = len(attrs)
    values = [np.zeros_like(a) for a in attrs]
    rows = [np.zeros(MAX_LODS, dtype=np.int8) for _ in attrs]
    IP = C.POINTER(C.c_int32) * k
    _check(lib().pccb200_attr_lift_encode_multi(
        C.byref(lod_params), C.c_int32(k), (C.POINTER(QpSet) * k)(*[C.pointer(q) for q in qpsets]),
        (C.c_int32 * k)(*[int(e) for e in (lcp_enabled or [0] * k)]), _p(xyz, C.c_int32),
        C.c_int32(xyz.shape[0]), IP(*[_p(a, C.c_int32) for a in attrs]),
        (C.c_int32 * k)(*[a.shape[1] for a in attrs]), (C.c_int32 * k)(*(bitdepths or [8] * k)),
        IP(*[_p(v, C.c_int32) for v in values]),
        (C.POINTER(C.c_int8) * k)(*[_p(r, C.c_int8) for r in rows])))
    return values, attrs, [r[:lod_params.num_detail_levels].copy() for r in rows]


def attr_lift_multi_decode(lod_params, qpsets, xyz, values, lcps=None, lcp_enabled=None,
                           bitdepths=None):
    """decoder counterpart of attr_lift_multi_encode: values[s] [N, A_s] (coding
    order), lcps[s] the encoder's lcp coefficients or None -> reconstruction[s]"""
    xyz = np.ascontiguousarray(xyz, dtype=np.int32)
    values = [np.ascontiguousarray(v, dtype=np.int32).reshape(xyz.shape[0], -1) for v in values]
    k = len(values)
    attrs = [np.zeros_like(v) for v in values]
    rows = [None] * k
    for s, l in enumerate(lcps or [None] * k):
        if l is not None:
            rows[s] = np.zeros(MAX_LODS, dtype=np.int8)
            rows[s][:len(l)] = l
    IP = C.POINTER(C.c_int32) * k
    _check(lib().pccb200_attr_lift_decode_multi(
        C.byref(lod_params), C.c_int32(k), (C.POINTER(QpSet) * k)(*[C.pointer(q) for q in qpsets]),
        (C.c_int32 * k)(*[int(e) for e in (lcp_enabled or [0] * k)]), _p(xyz, C.c_int32),
        C.c_int32(xyz.shape[0]), IP(*[_p(a, C.c_int32) for a in attrs]),
        (C.c_int32 * k)(*[v.shape[1] for v in values]), (C.c_int32 * k)(*(bitdepths or [8] * k)),
        IP(*[_p(v, C.c_int32) for v in values]),
        (C.POINTER(C.c_int8) * k)(*[_p(r, C.c_int8) for r in rows])))
    return attrs


def attr_lift_multi_batch_dev(forward, lods, qpsets, xyzs, attrs, values, lcps, lcp_enabled=None,
                              bitdepths=None):
    """as attr_lift_multi_batch with contiguous int32 torch CUDA tensors (device
    pointers): xyzs[u], attrs[u][s] (in and out when forward, out otherwise),
    values[u][s] (out when forward, in otherwise); lcps: host int8 numpy array
    [units, sets, MAX_LODS] (out when forward, in otherwise).  The producing
    stream must be synchronised before the call (see the header)."""
    tensors = list(xyzs) + [a for u in attrs for a in u] + [v for u in values for v in u]
    for t in tensors:
        if not (t.is_cuda and t.is_contiguous() and str(t.dtype) == "torch.int32"):
            raise PccB200Error("attr_lift_multi_batch_dev takes contiguous int32 CUDA tensors")
    if not (isinstance(lcps, np.ndarray) and lcps.dtype == np.int8 and lcps.flags.c_contiguous
            and lcps.shape == (len(xyzs), len(qpsets), MAX_LODS)):
        raise PccB200Error("lcps must be a contiguous int8 array [units, sets, MAX_LODS]")
    args = _lift_multi_args(lods, qpsets, lcp_enabled, xyzs, attrs, values,
                            [list(u) for u in lcps], bitdepths, lambda x: x.data_ptr())
    fn = (lib().pccb200_attr_lift_encode_multi_batch_dev if forward
          else lib().pccb200_attr_lift_decode_multi_batch_dev)
    _check(fn(*args))


def _scalable_args(scals, args):
    """a *_multi_batch argument tuple with the LodScalable array after lods"""
    return args[:2] + ((LodScalable * len(scals))(*scals),) + args[2:]


def attr_lift_scalable(forward, lods, scals, qpsets, xyzs, data, lcp_enabled=None,
                       bitdepths=None, lcps=None):
    """Scalable lifting (pccb200_attr_lift_{en,de}code_scalable), shaped as
    attr_lift_multi_batch with scals[u] the LodScalable of unit u.  lcp rows
    have SCALABLE_LODS entries."""
    xyzs = [np.ascontiguousarray(x, dtype=np.int32) for x in xyzs]
    data = [[np.ascontiguousarray(a, dtype=np.int32).reshape(x.shape[0], -1) for a in u]
            for x, u in zip(xyzs, data)]
    if forward:
        attrs = [[a.copy() for a in u] for u in data]
        values = [[np.zeros_like(a) for a in u] for u in data]
        rows = [[np.zeros(MAX_LODS, dtype=np.int8) for _ in u] for u in data]
    else:
        attrs = [[np.zeros_like(a) for a in u] for u in data]
        values = data
        rows = [[None] * len(u) for u in data]
        for u, lu in zip(rows, lcps if lcps is not None else []):
            for s, l in enumerate(lu if lu is not None else []):
                if l is not None:
                    u[s] = np.zeros(MAX_LODS, dtype=np.int8)
                    u[s][:len(l)] = l
    args = _lift_multi_args(lods, qpsets, lcp_enabled, xyzs, attrs, values, rows, bitdepths,
                            lambda x: x.ctypes.data)
    fn = (lib().pccb200_attr_lift_encode_scalable if forward
          else lib().pccb200_attr_lift_decode_scalable)
    _check(fn(*_scalable_args(scals, args)))
    if not forward:
        return attrs
    return values, attrs, [[r[:SCALABLE_LODS].copy() for r in u] for u in rows]


def attr_lift_scalable_dev(forward, lods, scals, qpsets, xyzs, attrs, values, lcps,
                           lcp_enabled=None, bitdepths=None):
    """as attr_lift_multi_batch_dev, for scalable lifting (scals[u] per unit)"""
    tensors = list(xyzs) + [a for u in attrs for a in u] + [v for u in values for v in u]
    for t in tensors:
        if not (t.is_cuda and t.is_contiguous() and str(t.dtype) == "torch.int32"):
            raise PccB200Error("attr_lift_scalable_dev takes contiguous int32 CUDA tensors")
    if not (isinstance(lcps, np.ndarray) and lcps.dtype == np.int8 and lcps.flags.c_contiguous
            and lcps.shape == (len(xyzs), len(qpsets), MAX_LODS)):
        raise PccB200Error("lcps must be a contiguous int8 array [units, sets, MAX_LODS]")
    args = _lift_multi_args(lods, qpsets, lcp_enabled, xyzs, attrs, values,
                            [list(u) for u in lcps], bitdepths, lambda x: x.data_ptr())
    fn = (lib().pccb200_attr_lift_encode_scalable_dev if forward
          else lib().pccb200_attr_lift_decode_scalable_dev)
    _check(fn(*_scalable_args(scals, args)))


def _i3(v):
    return (C.c_int32 * 3)(*[int(x) for x in v])


def xyz_to_rpl(laser_origin, laser_theta, xyz):
    """convertXyzToRpl -> (rpl [N,3], bbox (min[3], max[3]))"""
    xyz = np.ascontiguousarray(xyz, dtype=np.int32)
    theta = np.ascontiguousarray(laser_theta, dtype=np.int32)
    out = np.zeros_like(xyz)
    bbox = np.zeros(6, dtype=np.int32)
    _check(lib().pccb200_xyz_to_rpl(_i3(laser_origin), _p(theta, C.c_int32), C.c_int32(theta.size),
                                    _p(xyz, C.c_int32), C.c_int64(xyz.shape[0]),
                                    _p(out, C.c_int32), _p(bbox, C.c_int32)))
    return out, (bbox[:3].copy(), bbox[3:].copy())


def offset_and_scale(min_pos, axis_weight, pos):
    """offsetAndScale -> new positions [N,3]"""
    pos = np.ascontiguousarray(pos, dtype=np.int32).copy()
    _check(lib().pccb200_offset_and_scale(_i3(min_pos), _i3(axis_weight), _p(pos, C.c_int32),
                                          C.c_int64(pos.shape[0])))
    return pos


def attr_spherical_positions(laser_origin, laser_theta, axis_weight, xyz, min_pos=None):
    """conversion + offsetAndScale in one call -> (positions [N,3], bbox of the conversion)"""
    xyz = np.ascontiguousarray(xyz, dtype=np.int32)
    theta = np.ascontiguousarray(laser_theta, dtype=np.int32)
    out = np.zeros_like(xyz)
    bbox = np.zeros(6, dtype=np.int32)
    _check(lib().pccb200_attr_spherical_positions(
        _i3(laser_origin), _p(theta, C.c_int32), C.c_int32(theta.size), _i3(axis_weight),
        None if min_pos is None else _i3(min_pos), _p(xyz, C.c_int32), C.c_int64(xyz.shape[0]),
        _p(out, C.c_int32), _p(bbox, C.c_int32)))
    return out, (bbox[:3].copy(), bbox[3:].copy())


def coeff_symbols(coeffs):
    """planar coefficients [A, N] -> (zero_runs[S], values[S, A], ctx[S] or None, tail_run)"""
    coeffs = np.ascontiguousarray(coeffs, dtype=np.int32)
    a, n = coeffs.shape
    runs = np.zeros(n, dtype=np.int32)
    values = np.zeros((n, a), dtype=np.int32)
    ctx = np.zeros(n, dtype=np.uint8)
    cnt, tail = C.c_int32(0), C.c_int32(0)
    _check(lib().pccb200_coeff_symbols(_p(coeffs, C.c_int32), C.c_int32(a), C.c_int32(n),
                                       _p(runs, C.c_int32), _p(values, C.c_int32),
                                       _p(ctx, C.c_uint8), C.byref(cnt), C.byref(tail)))
    s = cnt.value
    return runs[:s].copy(), values[:s].copy(), (ctx[:s].copy() if a == 3 else None), tail.value


def attr_raht_encode_symbols(params, qpset, xyz, attrs, bitdepth=8, qpoffs=None):
    """-> (reconstruction [N, A], zero_runs, values, ctx, tail_run): the attribute
    encoder call handing over the entropy coder's symbol stream"""
    xyz = np.ascontiguousarray(xyz, dtype=np.int32)
    attrs = np.ascontiguousarray(attrs, dtype=np.int32).copy()
    n, a = attrs.shape
    runs = np.zeros(n, dtype=np.int32)
    values = np.zeros((n, a), dtype=np.int32)
    ctx = np.zeros(n, dtype=np.uint8)
    cnt, tail = C.c_int32(0), C.c_int32(0)
    if qpoffs is not None:
        qpoffs = np.ascontiguousarray(qpoffs, dtype=np.int32)
    _check(lib().pccb200_attr_raht_encode_symbols(
        C.byref(params), C.byref(qpset), _p(qpoffs, C.c_int32), _p(xyz, C.c_int32),
        _p(attrs, C.c_int32), C.c_int32(a), C.c_int32(n), C.c_int32(bitdepth),
        _p(runs, C.c_int32), _p(values, C.c_int32), _p(ctx, C.c_uint8), C.byref(cnt),
        C.byref(tail)))
    s = cnt.value
    return attrs, runs[:s].copy(), values[:s].copy(), (ctx[:s].copy() if a == 3 else None), tail.value


def estimate_dist2(xyz, sampling_period=100, search_range=128, percentile=0.85):
    """estimateDist2 -> shift bits"""
    xyz = np.ascontiguousarray(xyz, dtype=np.int32)
    out = C.c_int32(0)
    _check(lib().pccb200_estimate_dist2(_p(xyz, C.c_int32), C.c_int32(xyz.shape[0]),
                                        C.c_int32(sampling_period), C.c_int32(search_range),
                                        C.c_float(percentile), C.byref(out)))
    return out.value


def quant_weights_fixed(preds, num_points_in_lod, neigh_weight):
    """computeQuantizationWeights (predicting transform) -> qw[N]"""
    preds = np.ascontiguousarray(preds)
    npl = np.ascontiguousarray(num_points_in_lod, dtype=np.uint32)
    n = preds.shape[0]
    qw = np.zeros(n, dtype=np.uint64)
    _check(lib().pccb200_quant_weights_fixed(
        C.cast(preds.ctypes.data, C.POINTER(Predictor)), C.c_int32(n), _p(npl, C.c_uint32),
        C.c_int32(npl.size), _i3(neigh_weight), _p(qw, C.c_uint64)))
    return qw


def quant_weights_scalable(num_points_in_lod, num_points, min_geom_node_size_log2):
    """computeQuantizationWeightsScalable -> qw[N], N = num_points_in_lod[-1]"""
    npl = np.ascontiguousarray(num_points_in_lod, dtype=np.uint32)
    n = int(npl[-1])
    qw = np.zeros(n, dtype=np.uint64)
    _check(lib().pccb200_quant_weights_scalable(
        _p(npl, C.c_uint32), C.c_int32(npl.size), C.c_int64(num_points),
        C.c_int32(min_geom_node_size_log2), C.c_int32(n), _p(qw, C.c_uint64)))
    return qw

