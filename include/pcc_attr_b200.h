/* pcc_attr_b200.h — C ABI of the CUDA (H100) G-PCC attribute-transform path.
 *
 * Drop-in boundary for the attribute-transform hot path of MPEG G-PCC TMC13
 * (release-23.0-rc2).  Every entry point is `extern "C"`, takes plain host
 * pointers and sizes (no torch / C++ types) and returns an int status
 * (PCCB200_OK == 0).  The functions are synchronous: results are in the
 * caller's host buffers on return, mirroring the reference's own blocking
 * calls.
 *
 * Reference interfaces replaced (paths relative to the TMC13 tree):
 *   pccb200_raht_forward   <- pcc::regionAdaptiveHierarchicalTransform
 *                             tmc3/RAHT.h:47-57, tmc3/RAHT.cpp:1997-2018
 *   pccb200_raht_inverse   <- pcc::regionAdaptiveHierarchicalInverseTransform
 *                             tmc3/RAHT.h:59-69, tmc3/RAHT.cpp:2037-2058
 *   pccb200_morton_sort    <- mortonAddr + std::sort(MortonCodeWithIndex)
 *                             tmc3/AttributeEncoder.cpp:1316-1321,
 *                             tmc3/AttributeDecoder.cpp:623-628,
 *                             tmc3/PCCMath.h:605-626
 *   pccb200_attr_raht_encode / _decode
 *                          <- the sort + gather + transform + clip body of
 *                             AttributeEncoder::encode{Colors,Reflectances}TransformRaht
 *                             tmc3/AttributeEncoder.cpp:1214-1375 and
 *                             AttributeDecoder::decode{Colors,Reflectance}Raht
 *                             tmc3/AttributeDecoder.cpp:527-674 (entropy
 *                             coding stays on the host, in the caller)
 *   pccb200_quant_weights  <- pcc::PCCComputeQuantizationWeights
 *                             tmc3/PCCTMC3Common.h:828-854
 *   pccb200_lift_forward / _inverse
 *                          <- per-LoD PCCLiftPredict + PCCLiftUpdate loops
 *                             tmc3/AttributeEncoder.cpp:1408-1415,1476-1482,
 *                             tmc3/PCCTMC3Common.h:716-824
 *
 * Arithmetic is the reference's: Q.15 FixedPoint in int64 with
 * round-half-away multiplies (tmc3/FixedPoint.h:113-122), the LUT+Newton
 * isqrt/irsqrt (tmc3/misc.cpp:138-225) and the reciprocal-multiply Quantizer
 * (tmc3/quantization.h:79-102).  Outputs are bit-identical to the reference.
 */
#ifndef PCC_ATTR_B200_H
#define PCC_ATTR_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PCCB200_ABI_VERSION 1

/* status codes */
#define PCCB200_OK 0
#define PCCB200_ERR_INVALID_ARG 1   /* null pointer, bad size, A not in 1..3 */
#define PCCB200_ERR_NO_DEVICE 2     /* no CUDA device / wrong architecture */
#define PCCB200_ERR_CUDA 3          /* a CUDA runtime call failed */
#define PCCB200_ERR_UNSORTED 4      /* morton[] not ascending */
#define PCCB200_ERR_UNSUPPORTED 5   /* e.g. inter-frame prediction requested */
#define PCCB200_ERR_NOMEM 6

#define PCCB200_MAX_QP_LAYERS 32
#define PCCB200_MAX_AC_QP_LAYERS 32

/* Flattened pcc::RahtPredictionParams (tmc3/hls.h:439-466) plus the
 * `rahtExtension` bool argument of the transform entry points. */
typedef struct pccb200_raht_params {
  int32_t prediction_enabled;         /* raht_prediction_enabled_flag */
  int32_t integer_haar;               /* integer_haar_enable_flag */
  int32_t prediction_threshold0;      /* raht_prediction_threshold0 */
  int32_t prediction_threshold1;      /* raht_prediction_threshold1 */
  int32_t subnode_prediction_enabled; /* raht_subnode_prediction_enabled_flag */
  int32_t prediction_search_range;    /* raht_prediction_search_range */
  int32_t pred_weight_parent[19];     /* predWeightParent */
  int32_t pred_weight_child[12];      /* predWeightChild (used iff subnode) */
  int32_t raht_extension;             /* aps.raht_extension */
} pccb200_raht_params;

/* Flattened pcc::QpSet (tmc3/quantization.h:123-137).  Region offsets reach
 * the transform as per-point offsets (point_qp_offsets), exactly as in the
 * reference (tmc3/AttributeEncoder.cpp:1337). */
typedef struct pccb200_qpset {
  int32_t num_layers;                                  /* layers.size() >= 1 */
  int32_t layers[PCCB200_MAX_QP_LAYERS][2];            /* {luma, chroma offset} */
  int32_t max_qp;
  int32_t fixed_point_qp_offset;
  int32_t num_ac_coeff_qp_layers;                      /* rahtAcCoeffQps.size() */
  int32_t ac_coeff_qps[PCCB200_MAX_AC_QP_LAYERS][7][2];
} pccb200_qpset;

/* Fill p with the reference's defaults (tmc3/TMC3.cpp:1284-1318,
 * tmc3/hls.h:451-465): prediction on, thresholds 2/6, sub-node prediction on
 * with weights {9,3,1,5,2}, search range 50000, rahtExtension on. */
void pccb200_raht_params_default(pccb200_raht_params* p);

/* Derive the 19 + 12 prediction weights from the 5 signalled ones
 * (RahtPredictionParams::setPredictionWeights, tmc3/hls.h:456-465).
 * The reference normalises a prediction by a 64-entry reciprocal table indexed
 * by the sum of the weights that reached a child (tmc3/RAHT.cpp:445-451,
 * 567-570); a weight set with w[0] + 3*max(w[1],w[3]) + 3*max(w[2],w[4]) > 64
 * makes it read past that table.  This library evaluates the table's formula,
 * round(32768 / sum), for any sum: identical wherever the reference is defined. */
void pccb200_raht_set_prediction_weights(pccb200_raht_params* p,
                                         const int32_t w[5]);

/* Library / device management ------------------------------------------- */

int pccb200_abi_version(void);
/* Selects the CUDA device used by this process' calls (default 0). */
int pccb200_set_device(int device);
/* Human-readable description of the last error on this thread. */
const char* pccb200_last_error(void);
/* Number of kernel launches issued by this library since process start. */
uint64_t pccb200_kernel_launch_count(void);

/* Morton sort ------------------------------------------------------------ */

/* keys_out[i] = Morton code of the i-th point in ascending code order
 * (x -> bit 2, y -> bit 1, z -> bit 0 of each triple), ties kept in input
 * order; order_out[i] = its index in xyz.  xyz is N x 3 int32, coordinates in
 * [0, 2^21). */
int pccb200_morton_sort(const int32_t* xyz, int32_t n, int64_t* keys_out,
                        int32_t* order_out);

/* RAHT, reference-signature level ---------------------------------------- */

/* morton: N ascending codes.  attrs_inout: N x A row-major int32; in: source
 * values, out: reconstructed (unclipped) values.  coeffs_out: A x N planar.
 * point_qp_offsets: N x 2 int32 or NULL for all-zero. */
int pccb200_raht_forward(const pccb200_raht_params* params,
                         const pccb200_qpset* qpset,
                         const int32_t* point_qp_offsets,
                         const int64_t* morton, int32_t* attrs_inout,
                         int32_t num_attrs, int32_t n, int32_t* coeffs_out);

/* coeffs_in: A x N planar quantised coefficients.  attrs_out: N x A. */
int pccb200_raht_inverse(const pccb200_raht_params* params,
                         const pccb200_qpset* qpset,
                         const int32_t* point_qp_offsets,
                         const int64_t* morton, int32_t* attrs_out,
                         int32_t num_attrs, int32_t n,
                         const int32_t* coeffs_in);

/* RAHT, attribute-coder level (sort + gather + transform + clip on device) - */

/* xyz: N x 3 positions in input (unsorted) order.  attrs_inout: N x A values
 * in input order (uint16 range); on return the clipped reconstruction in
 * input order, as AttributeEncoder writes back into the PCCPointSet3.
 * coeffs_out: A x N planar, in coding order.  bitdepth gives the clip range
 * [0, 2^bitdepth - 1].  point_qp_offsets: N x 2 in input order, or NULL. */
int pccb200_attr_raht_encode(const pccb200_raht_params* params,
                             const pccb200_qpset* qpset,
                             const int32_t* point_qp_offsets,
                             const int32_t* xyz, int32_t* attrs_inout,
                             int32_t num_attrs, int32_t n, int32_t bitdepth,
                             int32_t* coeffs_out);

int pccb200_attr_raht_decode(const pccb200_raht_params* params,
                             const pccb200_qpset* qpset,
                             const int32_t* point_qp_offsets,
                             const int32_t* xyz, int32_t* attrs_out,
                             int32_t num_attrs, int32_t n, int32_t bitdepth,
                             const int32_t* coeffs_in);

/* Batched slices: the independent work units of a frame
 * (tmc3/encoder.cpp:545-568).  Slice s owns points
 * [slice_offsets[s], slice_offsets[s+1]) of every per-point array and the
 * matching range of every planar coefficient component:
 * coeffs[(k * total + slice_offsets[s]) ...] holds component k of slice s,
 * i.e. each slice's coefficients are planar with stride `total`. */
int pccb200_attr_raht_encode_slices(const pccb200_raht_params* params,
                                    const pccb200_qpset* qpset,
                                    const int32_t* point_qp_offsets,
                                    const int32_t* xyz, int32_t* attrs_inout,
                                    int32_t num_attrs, int32_t bitdepth,
                                    const int64_t* slice_offsets,
                                    int32_t num_slices, int32_t* coeffs_out);

/* Device-resident variants (inputs and outputs already in HBM) ------------- */

/* Calls made from different host threads run concurrently, each on its own
 * CUDA stream ("lane"); the slices of one *_slices call are spread over lanes
 * as well.  pccb200_time_begin() records a CUDA event that every lane waits
 * for, pccb200_time_end() one that waits for every lane, and returns the
 * elapsed device time between the two in milliseconds. */
int pccb200_time_begin(void);
int pccb200_time_end(double* ms_out);

/* As pccb200_attr_raht_encode_slices / a decode counterpart, but every array
 * pointer is a DEVICE pointer on the selected device; slice_offsets stays a
 * host array.
 *
 * Stream ordering: the library works on its own non-blocking streams, which
 * are NOT ordered with any stream of the caller.  Everything that produces
 * the input buffers must have completed before the call (synchronise the
 * producing stream, or an event recorded on it, first); the outputs are
 * complete when the call returns, so any stream may consume them afterwards.
 *
 * Concurrency: for calls from several host threads to overlap on the device
 * each lane needs its own hardware queue; set CUDA_DEVICE_MAX_CONNECTIONS=32
 * in the process environment before the CUDA context is created (with the
 * default of 8 a long dataflow kernel blocks the short kernels of a lane
 * that shares its queue).  The library does not touch the environment. */
int pccb200_attr_raht_encode_slices_dev(const pccb200_raht_params* params,
                                        const pccb200_qpset* qpset,
                                        const int32_t* d_point_qp_offsets,
                                        const int32_t* d_xyz,
                                        int32_t* d_attrs_inout, int32_t num_attrs,
                                        int32_t bitdepth,
                                        const int64_t* slice_offsets,
                                        int32_t num_slices,
                                        int32_t* d_coeffs_out);
int pccb200_attr_raht_decode_slices_dev(const pccb200_raht_params* params,
                                        const pccb200_qpset* qpset,
                                        const int32_t* d_point_qp_offsets,
                                        const int32_t* d_xyz, int32_t* d_attrs_out,
                                        int32_t num_attrs, int32_t bitdepth,
                                        const int64_t* slice_offsets,
                                        int32_t num_slices,
                                        const int32_t* d_coeffs_in);

/* Several attributes of one slice in ONE pass ----------------------------------
 *
 * The attributes of a slice are coded on the same positions
 * (tmc3/encoder.cpp:1052-1240 loops over them; AttributeEncoder::encode is
 * entered once per attribute): the Morton sort, the tree, the worklists, the
 * neighbour searches, the weights and, above all, the chain of block
 * dependencies are the same for all of them.  These entry points code up to
 * two attributes with at most four components together (typically colour +
 * reflectance): each keeps its own QpSet, coefficient planes and zero-run
 * state, and the results are bit-identical to one call per attribute.
 * Per-point qp offsets are not supported here (use the single-attribute
 * calls); parameter combinations without a fused path (AC-coefficient qp
 * offsets in the encoder) are coded attribute by attribute internally.
 *
 *   qpsets[s], attrs[s] (n x num_attrs[s], row-major, in/out), num_attrs[s],
 *   bitdepths[s], coeffs[s] (num_attrs[s] planes of n) describe attribute s.
 * The *_dev variants take device pointers for xyz, attrs[s] and coeffs[s]
 * (the pointer arrays themselves are host arrays); see the stream-ordering
 * note above. */
int pccb200_attr_raht_encode_multi(const pccb200_raht_params* params, int32_t num_sets,
                                   const pccb200_qpset* const* qpsets, const int32_t* xyz,
                                   int32_t* const* attrs_inout, const int32_t* num_attrs,
                                   const int32_t* bitdepths, int32_t n,
                                   int32_t* const* coeffs_out);
int pccb200_attr_raht_decode_multi(const pccb200_raht_params* params, int32_t num_sets,
                                   const pccb200_qpset* const* qpsets, const int32_t* xyz,
                                   int32_t* const* attrs_out, const int32_t* num_attrs,
                                   const int32_t* bitdepths, int32_t n,
                                   const int32_t* const* coeffs_in);
int pccb200_attr_raht_encode_multi_dev(const pccb200_raht_params* params, int32_t num_sets,
                                       const pccb200_qpset* const* qpsets,
                                       const int32_t* d_xyz, int32_t* const* d_attrs_inout,
                                       const int32_t* num_attrs, const int32_t* bitdepths,
                                       int32_t n, int32_t* const* d_coeffs_out);
int pccb200_attr_raht_decode_multi_dev(const pccb200_raht_params* params, int32_t num_sets,
                                       const pccb200_qpset* const* qpsets,
                                       const int32_t* d_xyz, int32_t* const* d_attrs_out,
                                       const int32_t* num_attrs, const int32_t* bitdepths,
                                       int32_t n, const int32_t* const* d_coeffs_in);

/* Many coding units in one call ----------------------------------------------
 *
 * The slices of a frame (tmc3/TMC3.cpp:781-810 cuts a frame into slices of at
 * most sliceMaxPoints points; tmc3/encoder.cpp:545-568 codes them one after
 * another) and the frames of a sequence are independent point sets.  A unit
 * whose coefficients are dense in small values is bound by the latency of its
 * own chain of blocks (the zero-run state of the encoder's RDOQ runs through
 * every coefficient in coding order, tmc3/RAHT.cpp:1154,1617-1670) and keeps
 * only a few warps busy: device throughput follows the number of units in
 * flight.  These entry points take num_units units with the same attributes
 * (num_sets, num_attrs[s], bitdepths[s], qpsets[s] as above) and code them in
 * gangs: the top-down passes of all units of a gang share their kernel
 * launches, so the units in flight are not limited by the number of streams.
 * Results are bit-identical to one pccb200_attr_raht_*_multi call per unit.
 *
 *   xyz[u] (n[u] x 3), attrs[u * num_sets + s] (n[u] x num_attrs[s], in/out),
 *   coeffs[u * num_sets + s] (num_attrs[s] planes of n[u]) describe unit u.
 * The pointer arrays are host arrays; in the *_dev variants their elements are
 * device pointers (stream-ordering note above).  Workspace: about 0.6 KB per
 * point and unit in flight. */
int pccb200_attr_raht_encode_multi_batch(const pccb200_raht_params* params, int32_t num_sets,
                                         const pccb200_qpset* const* qpsets, int32_t num_units,
                                         const int32_t* const* xyz, int32_t* const* attrs_inout,
                                         const int32_t* num_attrs, const int32_t* bitdepths,
                                         const int32_t* n, int32_t* const* coeffs_out);
int pccb200_attr_raht_decode_multi_batch(const pccb200_raht_params* params, int32_t num_sets,
                                         const pccb200_qpset* const* qpsets, int32_t num_units,
                                         const int32_t* const* xyz, int32_t* const* attrs_out,
                                         const int32_t* num_attrs, const int32_t* bitdepths,
                                         const int32_t* n, const int32_t* const* coeffs_in);
int pccb200_attr_raht_encode_multi_batch_dev(const pccb200_raht_params* params, int32_t num_sets,
                                             const pccb200_qpset* const* qpsets,
                                             int32_t num_units, const int32_t* const* d_xyz,
                                             int32_t* const* d_attrs_inout,
                                             const int32_t* num_attrs, const int32_t* bitdepths,
                                             const int32_t* n, int32_t* const* d_coeffs_out);
int pccb200_attr_raht_decode_multi_batch_dev(const pccb200_raht_params* params, int32_t num_sets,
                                             const pccb200_qpset* const* qpsets,
                                             int32_t num_units, const int32_t* const* d_xyz,
                                             int32_t* const* d_attrs_out,
                                             const int32_t* num_attrs, const int32_t* bitdepths,
                                             const int32_t* n, const int32_t* const* d_coeffs_in);

/* Recolouring: attribute transfer to the coded geometry ---------------------------
 *
 * When geometry coding adds or removes points (duplicate merging, lossy
 * quantisation, trisoup) the encoder transfers the attributes of the source
 * cloud onto the points it is going to code, right before attribute coding
 * (tmc3/encoder.cpp:1031-1037; recolour / recolourColour / recolourReflectance,
 * tmc3/pointset_processing.cpp:253-958).  For every target point: the
 * num_neighbours_fwd nearest source points give a (distance-weighted) forward
 * colour; the source points that have the target among their
 * num_neighbours_bwd nearest targets give a backward centroid; the result is
 * the colour within +-search_range of that centroid that minimises the larger
 * of the two squared errors.  Positions relate by
 *     posInTgt = posInSrc * source_to_target_scale - tgt_to_src_offset.
 *
 * The reference searches with nanoflann kd-trees; here both searches are exact
 * k-nearest-neighbour queries over a grid hash (see csrc/recolour.cuh), double
 * precision, the reference's operation order.  Ties in distance are broken by
 * the lower point index -- nanoflann's choice among equidistant candidates
 * depends on its tree traversal -- so the result is bit-exact against the
 * oracle (same rule) and equal to the compiled reference except where a tie
 * reaches the k-th neighbour (tests/test_recolour.py states the tolerance).
 * Coordinates must lie in [0, 2^21).  num_attrs is 3 (colour) or 1
 * (reflectance); attrs are N x num_attrs, row-major.  Fields mirror
 * RecolourParams (tmc3/pointset_processing.h:47-63); defaults =
 * tmc3/TMC3.cpp:1500-1551. */
typedef struct pccb200_recolour_params {
  double dist_offset_fwd;            /* 4 */
  double dist_offset_bwd;            /* 4 */
  double max_geometry_dist2_fwd;     /* 1000 (>= 512: unlimited) */
  double max_geometry_dist2_bwd;     /* 1000 */
  double max_attribute_dist2_fwd;    /* 1000 */
  double max_attribute_dist2_bwd;    /* 1000 */
  int32_t search_range;              /* 1 */
  int32_t num_neighbours_fwd;        /* 8 (<= 16) */
  int32_t num_neighbours_bwd;        /* 1 (<= 16) */
  int32_t use_dist_weighted_avg_fwd; /* 1 */
  int32_t use_dist_weighted_avg_bwd; /* 1 */
  int32_t skip_avg_if_identical_source_point_present_fwd; /* 1 */
  int32_t skip_avg_if_identical_source_point_present_bwd; /* 0 */
  int32_t reserved;
} pccb200_recolour_params;

void pccb200_recolour_params_default(pccb200_recolour_params* p);

/* Host pointers.  target_attrs_out: n_target x num_attrs. */
int pccb200_recolour(const pccb200_recolour_params* params, const int32_t* source_xyz,
                     const int32_t* source_attrs, int32_t num_attrs, int32_t n_source,
                     double source_to_target_scale, const int32_t tgt_to_src_offset[3],
                     const int32_t* target_xyz, int32_t n_target, int32_t bitdepth,
                     int32_t* target_attrs_out);

/* Several attribute sets of a slice in one call, and many slices or frames --
 *
 * The encoder recolours every attribute of a slice onto the same coded
 * positions (tmc3/encoder.cpp:1031-1037 calls recolour() once per attribute;
 * recolourColour and recolourReflectance, tmc3/pointset_processing.cpp:253-958,
 * each build both kd-trees and run both searches).  None of that depends on the
 * attribute values, so these entries do it once per unit: both grid hashes,
 * the forward and backward k-nearest-neighbour searches, the backward lists
 * and their sort.  The forward and final colours of all num_sets sets (1 to
 * PCCB200_MAX_RECOLOUR_SETS) are then computed together, one launch each; a
 * call launches as many kernels for two sets as for one.  Each set's output is
 * bit-identical to one pccb200_recolour call per set, and so to the oracle.
 *
 *   source_attrs[s] (n_source x num_attrs[s]), num_attrs[s] (1 or 3),
 *   bitdepths[s] (1..16), target_attrs_out[s] (n_target x num_attrs[s])
 *   describe set s.
 *
 * The *_batch entries take num_units units (the slices of a frame, or whole
 * frames): source_xyz[u] (n_source[u] x 3), target_xyz[u] (n_target[u] x 3),
 * source_attrs[u * num_sets + s] and target_attrs_out[u * num_sets + s] as
 * above.  Scale and offset are per unit (source_to_target_scale[u],
 * tgt_to_src_offsets[3 * u .. 3 * u + 2]) because the slices of a frame differ
 * in their origin (_sliceOrigin).  Units are spread over the library's lanes;
 * results are bit-identical to one pccb200_recolour_multi call per unit.
 *
 * The *_dev entries take device pointers for positions and attributes; the
 * pointer arrays, num_attrs, bitdepths, scales and offsets stay host arrays.
 * The stream-ordering note of the RAHT *_dev entries applies.
 *
 * Arguments are checked before a device is looked up; every malformed one
 * returns PCCB200_ERR_INVALID_ARG.  A coordinate outside [0, 2^21) is found on
 * the device: PCCB200_ERR_INVALID_ARG, and pccb200_last_error() names the unit.
 *
 * Workspace of a unit in flight, with kf = num_neighbours_fwd, kb =
 * num_neighbours_bwd and SA = the sum of num_attrs[s]: 36 + 24 kb bytes per
 * source point and 44 + 12 kf + 4 SA bytes per target point, plus 12 bytes per
 * point and cell-size attempt of each grid's sort (usually two to four
 * attempts); the host-pointer entries add 12 + 4 SA bytes per point on either
 * side for the staged copies.  With the defaults (8 / 1 neighbours) and colour
 * plus reflectance: about 0.2 KB per target point and 0.1 KB per source point. */
#define PCCB200_MAX_RECOLOUR_SETS 4
int pccb200_recolour_multi(const pccb200_recolour_params* params, int32_t num_sets,
                           const int32_t* source_xyz, int32_t n_source,
                           const int32_t* const* source_attrs, const int32_t* num_attrs,
                           const int32_t* bitdepths, double source_to_target_scale,
                           const int32_t tgt_to_src_offset[3],
                           const int32_t* target_xyz, int32_t n_target,
                           int32_t* const* target_attrs_out);
int pccb200_recolour_multi_dev(const pccb200_recolour_params* params, int32_t num_sets,
                               const int32_t* d_source_xyz, int32_t n_source,
                               const int32_t* const* d_source_attrs, const int32_t* num_attrs,
                               const int32_t* bitdepths, double source_to_target_scale,
                               const int32_t tgt_to_src_offset[3],
                               const int32_t* d_target_xyz, int32_t n_target,
                               int32_t* const* d_target_attrs_out);
int pccb200_recolour_multi_batch(const pccb200_recolour_params* params, int32_t num_sets,
                                 int32_t num_units,
                                 const int32_t* const* source_xyz, const int32_t* n_source,
                                 const int32_t* const* source_attrs,
                                 const int32_t* num_attrs, const int32_t* bitdepths,
                                 const double* source_to_target_scale,
                                 const int32_t* tgt_to_src_offsets,
                                 const int32_t* const* target_xyz, const int32_t* n_target,
                                 int32_t* const* target_attrs_out);
int pccb200_recolour_multi_batch_dev(const pccb200_recolour_params* params, int32_t num_sets,
                                     int32_t num_units,
                                     const int32_t* const* d_source_xyz, const int32_t* n_source,
                                     const int32_t* const* d_source_attrs,
                                     const int32_t* num_attrs, const int32_t* bitdepths,
                                     const double* source_to_target_scale,
                                     const int32_t* tgt_to_src_offsets,
                                     const int32_t* const* d_target_xyz, const int32_t* n_target,
                                     int32_t* const* d_target_attrs_out);

/* Reference-exact recolouring --
 *
 * The entries above find their neighbours over a grid hash and break distance
 * ties by the lower point index.  These find them as the reference encoder
 * does: they build the kd-tree nanoflann builds for
 * KDTreeVectorOfVectorsAdaptor<PCCPointSet3, double> (metric_L2, leaf size 10),
 * on the device, level by level, and run nanoflann's findNeighbors on it, one
 * thread per query, with the same arithmetic; among equidistant candidates the
 * one nanoflann's traversal meets first is kept, as in the reference.  Each
 * target's backward list is put in the order libstdc++'s std::sort (g++ 13)
 * leaves it, which decides the order of the sums that follow.  The result
 * equals recolourColour / recolourReflectance (tmc3/pointset_processing.cpp)
 * bit for bit, ties, duplicate points and non-dyadic scales included.  The
 * two families differ on purpose wherever a distance tie reaches the k-th
 * neighbour.
 *
 * Same arguments and same rules as pccb200_recolour,
 * pccb200_recolour_multi_batch and pccb200_recolour_multi_batch_dev, except
 * the coordinate range: any int32 coordinate and offset of |x| < 2^30 (so that
 * target + offset cannot overflow); one outside it returns
 * PCCB200_ERR_INVALID_ARG, found on the device.  The other arguments are
 * checked before any device lookup.  The position-only work (both trees, both
 * searches, the backward lists) runs once per unit for all sets.
 *
 * Workspace of a unit in flight: up to about 300 bytes per point on either
 * side for the two trees and their build, on top of the lists of the entries
 * above. */
int pccb200_recolour_exact(const pccb200_recolour_params* params, const int32_t* source_xyz,
                           const int32_t* source_attrs, int32_t num_attrs, int32_t n_source,
                           double source_to_target_scale, const int32_t tgt_to_src_offset[3],
                           const int32_t* target_xyz, int32_t n_target, int32_t bitdepth,
                           int32_t* target_attrs_out);
int pccb200_recolour_exact_multi_batch(const pccb200_recolour_params* params, int32_t num_sets,
                                       int32_t num_units,
                                       const int32_t* const* source_xyz, const int32_t* n_source,
                                       const int32_t* const* source_attrs,
                                       const int32_t* num_attrs, const int32_t* bitdepths,
                                       const double* source_to_target_scale,
                                       const int32_t* tgt_to_src_offsets,
                                       const int32_t* const* target_xyz, const int32_t* n_target,
                                       int32_t* const* target_attrs_out);
int pccb200_recolour_exact_multi_batch_dev(const pccb200_recolour_params* params,
                                           int32_t num_sets, int32_t num_units,
                                           const int32_t* const* d_source_xyz,
                                           const int32_t* n_source,
                                           const int32_t* const* d_source_attrs,
                                           const int32_t* num_attrs, const int32_t* bitdepths,
                                           const double* source_to_target_scale,
                                           const int32_t* tgt_to_src_offsets,
                                           const int32_t* const* d_target_xyz,
                                           const int32_t* n_target,
                                           int32_t* const* d_target_attrs_out);

/* Per-phase device timing (CUDA events around every kernel launch on
 * the call's stream).  Phases: 0 Morton keys + radix sort, 1 tree build
 * (histogram, compaction, leaf / merge kernels), 2 block transform (the
 * top-down dataflow kernels), 3 duplicate tail + write-back, 4 gather /
 * scatter / clip, 5 lifting passes, 6 block geometry (worklists, neighbour
 * searches, qp descent: shared by everything that codes the same positions),
 * 7 block schedule (dependency levels + sort into wavefront order).
 * pccb200_profile_read returns the accumulated milliseconds and launch
 * counts since the last reset. */
#define PCCB200_NUM_PHASES 8
void pccb200_profile_enable(int enable);
void pccb200_profile_reset(void);
void pccb200_profile_read(double ms_out[PCCB200_NUM_PHASES],
                          uint64_t launches_out[PCCB200_NUM_PHASES]);

/* Lifting transform ------------------------------------------------------- */

/* Flattened pcc::PCCPredictor as consumed by the lifting passes
 * (tmc3/PCCTMC3Common.h:521-712): up to 3 neighbours, 8-bit fixed-point
 * weights, neighbour given as predictor index. */
typedef struct pccb200_predictor {
  uint32_t neighbor_count;
  uint32_t predictor_index[3];
  uint32_t weight[3];
} pccb200_predictor;

/* Flattened LoD-relevant fields of pcc::AttributeParameterSet
 * (tmc3/hls.h:795-857) plus abh.attr_dist2_delta.  Intra coding, default
 * point order; scalable lifting adds a pccb200_lod_scalable. */
#define PCCB200_MAX_LODS 32
typedef struct pccb200_lod_params {
  int32_t num_detail_levels;         /* num_detail_levels_minus1 + 1 */
  int32_t lod_decimation_type;       /* 0 distance, 1 periodic, 2 centroid */
  int32_t lod_sampling_period[PCCB200_MAX_LODS];
  int32_t dist2;                     /* aps.dist2 + abh.attr_dist2_delta */
  int32_t num_pred_nearest_neighbours; /* ..._minus1 + 1, 1..3 */
  int32_t inter_lod_search_range;
  int32_t intra_lod_search_range;
  int32_t intra_lod_prediction_skip_layers; /* >= num_detail_levels: none */
  int32_t prediction_with_distribution;
  int32_t lod_neigh_bias[3];
  int32_t pred_weight_blending;      /* predicting transform only */
} pccb200_lod_params;

/* Scalable lifting (aps.scalable_lifting_enabled_flag, lifting transform only),
 * given beside a pccb200_lod_params.  The levels of detail are the octree
 * levels: level l keeps, per octree node of size 2^(l+1), the point nearest to
 * the node's centroid, and neighbours farther than max_neigh_range at that
 * level are pruned (tmc3/PCCTMC3Common.h:2150-2235, :1918-1937, :2377-2446).
 * With it, num_detail_levels and dist2 of the pccb200_lod_params are not read;
 * lod_decimation_type must be 0.
 *   max_neigh_range          aps.max_neigh_range_minus1 + 1, >= 1
 *   min_geom_node_size_log2  first level: 0, or the octree level where a
 *                            partial geometry decode stopped (--decodeMaxPoints)
 *   geom_num_points          geom_num_points_minus1 + 1 of the slice, >= n; 0
 *                            means n (the encoder, and every full decode)
 *   reserved                 0 */
typedef struct pccb200_lod_scalable {
  int32_t max_neigh_range;
  int32_t min_geom_node_size_log2;
  int64_t geom_num_points;
  int32_t reserved;
} pccb200_lod_scalable;

/* Level-of-detail build: AttributeLods::generate (tmc3/AttributeCommon.cpp:45-72)
 * = buildPredictorsFast (tmc3/PCCTMC3Common.h:2300-2469: Morton sort,
 * subsampling, the atlas / window nearest-neighbour search, updatePredictors)
 * + PCCPredictor::computeWeights (+ blendWeights).
 * xyz: N x 3 positions.  preds_out[N] in predictor order (coarse to fine),
 * indexes_out[N]: predictor order -> point index, num_points_in_lod_out
 * [PCCB200_MAX_LODS]: cumulative LoD sizes, *lod_count_out their number. */
int pccb200_lod_build(const pccb200_lod_params* params, const int32_t* xyz,
                      int32_t n, pccb200_predictor* preds_out,
                      uint32_t* indexes_out, uint32_t* num_points_in_lod_out,
                      int32_t* lod_count_out);
/* The same for scalable lifting (AttributeLods::generate with
 * scalable_lifting_enabled_flag and minGeomNodeSizeLog2 =
 * scal->min_geom_node_size_log2).  At most 21 levels of detail. */
int pccb200_lod_build_scalable(const pccb200_lod_params* params,
                               const pccb200_lod_scalable* scal, const int32_t* xyz,
                               int32_t n, pccb200_predictor* preds_out,
                               uint32_t* indexes_out, uint32_t* num_points_in_lod_out,
                               int32_t* lod_count_out);

/* qw_out[i] for i in [0, n): PCCComputeQuantizationWeights. */
int pccb200_quant_weights(const pccb200_predictor* preds, int32_t n,
                          const uint32_t* num_points_in_lod, int32_t lod_count,
                          uint64_t* qw_out);

/* computeQuantizationWeights (tmc3/PCCTMC3Common.h:895-921, predicting
 * transform): the same walk with the per-slot weights neigh_weight[3]
 * (aps.quant_neigh_weight) instead of the predictors' own. */
int pccb200_quant_weights_fixed(const pccb200_predictor* preds, int32_t n,
                                const uint32_t* num_points_in_lod, int32_t lod_count,
                                const int32_t neigh_weight[3], uint64_t* qw_out);
/* computeQuantizationWeightsScalable (tmc3/PCCTMC3Common.h:858-891). */
int pccb200_quant_weights_scalable(const uint32_t* num_points_in_lod, int32_t lod_count,
                                   int64_t num_points, int32_t min_geom_node_size_log2,
                                   int32_t n, uint64_t* qw_out);

/* attrs_inout: N x A int64 in predictor order (values already << 8).
 * Forward: for lod = lod_count-1 .. 1: predict then update
 * (tmc3/AttributeEncoder.cpp:1408-1415).  Inverse: lod = 1 .. lod_count-1:
 * update then predict (tmc3/AttributeEncoder.cpp:1476-1482). */
int pccb200_lift_forward(const pccb200_predictor* preds, const uint64_t* qw,
                         int32_t n, const uint32_t* num_points_in_lod,
                         int32_t lod_count, int64_t* attrs_inout,
                         int32_t num_attrs);
int pccb200_lift_inverse(const pccb200_predictor* preds, const uint64_t* qw,
                         int32_t n, const uint32_t* num_points_in_lod,
                         int32_t lod_count, int64_t* attrs_inout,
                         int32_t num_attrs);

/* Lifting quantisation (+ last-component prediction) of the coefficients in
 * predictor order: the per-coefficient arithmetic of
 * tmc3/AttributeEncoder.cpp:1424-1473,1597-1625 and
 * computeLastComponentPredictionCoeff (:1498-1539).  attrs_inout: N x A
 * lifting coefficients in, reconstructed coefficients out.  values_out: N x A
 * quantised values (what the reference hands to its entropy coder).
 * lcp_coeffs_out: num_detail_levels entries (colour with lcp_enabled), may be
 * NULL otherwise.  point_qp_offsets: N x 2 in predictor order, or NULL.
 * qpset.fixed_point_qp_offset must carry the lifting offset (24,
 * tmc3/quantization.cpp:160-163). */
int pccb200_lift_quantize(const pccb200_qpset* qpset,
                          const int32_t* point_qp_offsets, const uint64_t* qw,
                          int32_t n, const uint32_t* num_points_in_lod,
                          int32_t lod_count, int32_t num_detail_levels,
                          int64_t* attrs_inout, int32_t num_attrs,
                          int32_t lcp_enabled, int32_t* values_out,
                          int8_t* lcp_coeffs_out);
/* Decoder side (tmc3/AttributeDecoder.cpp:711-749,815-837): values -> coefficients. */
int pccb200_lift_dequantize(const pccb200_qpset* qpset,
                            const int32_t* point_qp_offsets, const uint64_t* qw,
                            int32_t n, const uint32_t* num_points_in_lod,
                            int32_t lod_count, int32_t num_detail_levels,
                            const int32_t* values_in, int32_t num_attrs,
                            const int8_t* lcp_coeffs, int64_t* attrs_out);

/* The lifting attribute coder without its entropy coding, entirely on the
 * device (AttributeEncoder::encode{Colors,Reflectances}Lift,
 * tmc3/AttributeEncoder.cpp:1379-1494,1543-1648): LoD build, quantisation
 * weights, forward lifting, LCP + quantisation, inverse lifting, clip.
 * attrs_inout: N x A in input order, overwritten with the reconstruction.
 * values_out: N x A in coding (predictor) order.  point_qp_offsets: input
 * order or NULL.  lcp_coeffs_out: num_detail_levels entries or NULL. */
int pccb200_attr_lift_encode(const pccb200_lod_params* lod,
                             const pccb200_qpset* qpset, int32_t lcp_enabled,
                             const int32_t* point_qp_offsets, const int32_t* xyz,
                             int32_t* attrs_inout, int32_t num_attrs, int32_t n,
                             int32_t bitdepth, int32_t* values_out,
                             int8_t* lcp_coeffs_out);
/* Decoder counterpart (AttributeDecoder::decode{Colors,Reflectances}Lift). */
int pccb200_attr_lift_decode(const pccb200_lod_params* lod,
                             const pccb200_qpset* qpset, int32_t lcp_enabled,
                             const int32_t* point_qp_offsets, const int32_t* xyz,
                             int32_t* attrs_out, int32_t num_attrs, int32_t n,
                             int32_t bitdepth, const int32_t* values_in,
                             const int8_t* lcp_coeffs);

/* The slices of a frame, each with its own levels of detail, each on its own
 * lane (they overlap on the device).  Slice s owns points
 * [slice_offsets[s], slice_offsets[s+1]) of every per-point array and row s
 * (PCCB200_MAX_LODS entries) of the lcp array. */
int pccb200_attr_lift_encode_slices(const pccb200_lod_params* lod, const pccb200_qpset* qpset,
                                    int32_t lcp_enabled, const int32_t* point_qp_offsets,
                                    const int32_t* xyz, int32_t* attrs_inout,
                                    int32_t num_attrs, int32_t bitdepth,
                                    const int64_t* slice_offsets, int32_t num_slices,
                                    int32_t* values_out, int8_t* lcp_coeffs_out);
int pccb200_attr_lift_decode_slices(const pccb200_lod_params* lod, const pccb200_qpset* qpset,
                                    int32_t lcp_enabled, const int32_t* point_qp_offsets,
                                    const int32_t* xyz, int32_t* attrs_out, int32_t num_attrs,
                                    int32_t bitdepth, const int64_t* slice_offsets,
                                    int32_t num_slices, const int32_t* values_in,
                                    const int8_t* lcp_coeffs);

/* The same with device pointers for point_qp_offsets, xyz, attrs (coded in
 * place) and values (slice_offsets and the lcp coefficients stay host arrays);
 * stream-ordering note as for the RAHT *_dev entries. */
int pccb200_attr_lift_encode_slices_dev(const pccb200_lod_params* lod, const pccb200_qpset* qpset,
                                        int32_t lcp_enabled, const int32_t* d_point_qp_offsets,
                                        const int32_t* d_xyz, int32_t* d_attrs_inout,
                                        int32_t num_attrs, int32_t bitdepth,
                                        const int64_t* slice_offsets, int32_t num_slices,
                                        int32_t* d_values_out, int8_t* lcp_coeffs_out);
int pccb200_attr_lift_decode_slices_dev(const pccb200_lod_params* lod, const pccb200_qpset* qpset,
                                        int32_t lcp_enabled, const int32_t* d_point_qp_offsets,
                                        const int32_t* d_xyz, int32_t* d_attrs_out,
                                        int32_t num_attrs, int32_t bitdepth,
                                        const int64_t* slice_offsets, int32_t num_slices,
                                        const int32_t* d_values_in, const int8_t* lcp_coeffs);

/* Levels of detail kept across the attributes of a slice ------------------------
 *
 * AttributeEncoder / AttributeDecoder keep the LoDs of a slice
 * (tmc3/AttributeEncoder.h:183 `_lods`) and rebuild them only when the next
 * attribute's parameters differ (AttributeLods::isReusable,
 * tmc3/AttributeCommon.cpp:76-140; caller tmc3/encoder.cpp:1209-1210).  The
 * handle owns the device-resident predictors, the predictor order and the
 * quantisation weights of one slice; the colour call and the reflectance
 * call of the slice then run the lifting passes only. */
typedef struct pccb200_lod_handle_s* pccb200_lod_handle;

/* Builds the levels of detail of xyz (N x 3, host) on the selected device:
 * predictors and coding order.  The lifting quantisation weights are computed
 * by the first pccb200_attr_lift_*_lod call on the handle (a handle made for the
 * predicting transform, whose predictors reference their own level of detail,
 * never needs them). */
int pccb200_lod_create(const pccb200_lod_params* params, const int32_t* xyz, int32_t n,
                       pccb200_lod_handle* handle_out);
/* A handle over levels of detail the caller already holds (pcc::AttributeLods
 * after AttributeLods::generate, whoever built them), so that the lifting entries
 * below code on them unchanged.
 *   preds[n], indexes[n]   predictor order, as pccb200_lod_build returns them
 *   num_points_in_lod      lod_count cumulative counts, the last one n
 *   num_detail_levels      aps.maxNumDetailLevels(): the length of the LCP rows
 *                          (num_detail_levels_minus1 + 1, or 21 with scalable
 *                          lifting); lod_count..PCCB200_MAX_LODS
 *   scal                   NULL, or scalable lifting: the quantisation weights are
 *                          then computeQuantizationWeightsScalable with
 *                          (geom_num_points, min_geom_node_size_log2) of scal, the
 *                          encoder's (0 or n, 0) or the decoder's; max_neigh_range
 *                          is not read
 * Host checks, before any device lookup, return PCCB200_ERR_INVALID_ARG: null
 * pointers, n <= 0, lod_count outside 1..PCCB200_MAX_LODS, counts that decrease
 * (equal neighbours are an empty level, which the reference's scalable levels
 * have) or start at 0, a last count other than n, num_detail_levels out of
 * range, and a malformed scal.  On the device: indexes that are not a
 * permutation of [0, n), or a predictor with more than three neighbours or one
 * outside [0, n), return PCCB200_ERR_INVALID_ARG too.  Predictors that reference
 * their own level of detail are refused by the lifting calls
 * (PCCB200_ERR_UNSUPPORTED).  pccb200_lod_reusable is 0 for such a handle. */
int pccb200_lod_import(const pccb200_predictor* preds, const uint32_t* indexes, int32_t n,
                       const uint32_t* num_points_in_lod, int32_t lod_count,
                       int32_t num_detail_levels, const pccb200_lod_scalable* scal,
                       pccb200_lod_handle* handle_out);
void pccb200_lod_destroy(pccb200_lod_handle handle);
/* 1 if LoDs built with the handle's parameters serve `params` as well (the
 * comparisons of AttributeLods::isReusable that this structure carries), else 0. */
int pccb200_lod_reusable(pccb200_lod_handle handle, const pccb200_lod_params* params);
/* number of points / of LoDs; num_points_in_lod_out: PCCB200_MAX_LODS entries or NULL */
int pccb200_lod_info(pccb200_lod_handle handle, int32_t* n_out, int32_t* lod_count_out,
                     uint32_t* num_points_in_lod_out);
/* As pccb200_attr_lift_encode / _decode without positions and LoD
 * parameters: the handle's. */
int pccb200_attr_lift_encode_lod(pccb200_lod_handle handle, const pccb200_qpset* qpset,
                                 int32_t lcp_enabled, const int32_t* point_qp_offsets,
                                 int32_t* attrs_inout, int32_t num_attrs, int32_t bitdepth,
                                 int32_t* values_out, int8_t* lcp_coeffs_out);
int pccb200_attr_lift_decode_lod(pccb200_lod_handle handle, const pccb200_qpset* qpset,
                                 int32_t lcp_enabled, const int32_t* point_qp_offsets,
                                 int32_t* attrs_out, int32_t num_attrs, int32_t bitdepth,
                                 const int32_t* values_in, const int8_t* lcp_coeffs);

/* Several attributes of one slice in ONE lifting pass ---------------------------
 *
 * For attributes that share the positions and the LoD parameters of a slice --
 * the case where the reference reuses _lods for the next attribute
 * (AttributeLods::isReusable) -- these entries build the levels of detail and
 * the quantisation weights once, and run the forward and inverse lifting
 * passes once over the components of all num_sets sets (1 to
 * PCCB200_MAX_LIFT_SETS) side by side: a call makes the lifting-pass launches
 * of one attribute whatever the number of sets.  Each set keeps its own QpSet,
 * last-component prediction, bit-depth clip and outputs, and its results are
 * bit-identical to one pccb200_attr_lift_encode / _decode call per set.
 * Attributes whose LoD parameters differ need separate calls.  Per-point qp
 * offsets are not taken here (use the one-attribute entries).
 *
 *   qpsets[s], lcp_enabled[s], attrs[s] (n x num_attrs[s], point order; in and
 *   out when encoding, out when decoding), num_attrs[s] (1 or 3), bitdepths[s]
 *   (1..16), values[s] (n x num_attrs[s], coding order) and lcp_coeffs[s] (a
 *   host row of PCCB200_MAX_LODS entries, num_detail_levels of them used)
 *   describe set s.  lcp_coeffs[s] may be NULL where the set does not use it
 *   (the decoder needs it for a three-component set with lcp_enabled; the
 *   encoder writes it when given), and lcp_coeffs itself may be NULL when no
 *   set does.
 *
 * The *_batch entries take num_units units (the slices of a frame, or whole
 * frames), each with its own LoD parameters lods[u] (dist2 is set per slice,
 * abh.attr_dist2_delta), positions xyz[u] (n[u] x 3) and per set
 * attrs[u * num_sets + s], values[u * num_sets + s] and
 * lcp_coeffs[u * num_sets + s]; qpsets, lcp_enabled, num_attrs and bitdepths
 * are per set.  Units are spread over the library's lanes; results are
 * bit-identical to one *_multi call per unit.
 *
 * The *_dev entries take device pointers for positions, attributes and values;
 * the pointer arrays, the lcp rows and every per-set scalar stay on the host.
 * The stream-ordering note of the RAHT *_dev entries applies.
 *
 * Arguments are checked before a device is looked up; every malformed one
 * returns PCCB200_ERR_INVALID_ARG, and pccb200_last_error() names the unit or
 * the set.  Predictors that reference their own level of detail return
 * PCCB200_ERR_UNSUPPORTED, as the one-attribute entries do.
 *
 * Workspace of a unit in flight, with SA = the sum of num_attrs[s].  This is
 * an estimate summed from the per-point allocations of the LoD build, the
 * predictors, the quantisation weights and the lifting coefficients; it has not
 * been measured.  About 160 bytes per point for the levels of detail and the
 * quantisation weights (plus 4 ceil(log2 n) with centroid decimation, and the
 * grid-cell tables), and at most 8 + 16 SA for the lifting.  The host-pointer
 * entries add 12 + 12 SA for the staged copies.  Colour plus reflectance: about
 * 0.23 KB per point, 0.29 KB with host pointers. */
#define PCCB200_MAX_LIFT_SETS 4
int pccb200_attr_lift_encode_multi(const pccb200_lod_params* lod, int32_t num_sets,
                                   const pccb200_qpset* const* qpsets, const int32_t* lcp_enabled,
                                   const int32_t* xyz, int32_t n, int32_t* const* attrs_inout,
                                   const int32_t* num_attrs, const int32_t* bitdepths,
                                   int32_t* const* values_out, int8_t* const* lcp_coeffs_out);
int pccb200_attr_lift_decode_multi(const pccb200_lod_params* lod, int32_t num_sets,
                                   const pccb200_qpset* const* qpsets, const int32_t* lcp_enabled,
                                   const int32_t* xyz, int32_t n, int32_t* const* attrs_out,
                                   const int32_t* num_attrs, const int32_t* bitdepths,
                                   const int32_t* const* values_in,
                                   const int8_t* const* lcp_coeffs);
int pccb200_attr_lift_encode_multi_dev(const pccb200_lod_params* lod, int32_t num_sets,
                                       const pccb200_qpset* const* qpsets,
                                       const int32_t* lcp_enabled, const int32_t* d_xyz,
                                       int32_t n, int32_t* const* d_attrs_inout,
                                       const int32_t* num_attrs, const int32_t* bitdepths,
                                       int32_t* const* d_values_out,
                                       int8_t* const* lcp_coeffs_out);
int pccb200_attr_lift_decode_multi_dev(const pccb200_lod_params* lod, int32_t num_sets,
                                       const pccb200_qpset* const* qpsets,
                                       const int32_t* lcp_enabled, const int32_t* d_xyz,
                                       int32_t n, int32_t* const* d_attrs_out,
                                       const int32_t* num_attrs, const int32_t* bitdepths,
                                       const int32_t* const* d_values_in,
                                       const int8_t* const* lcp_coeffs);
int pccb200_attr_lift_encode_multi_batch(int32_t num_units, const pccb200_lod_params* const* lods,
                                         int32_t num_sets, const pccb200_qpset* const* qpsets,
                                         const int32_t* lcp_enabled, const int32_t* const* xyz,
                                         const int32_t* n, int32_t* const* attrs_inout,
                                         const int32_t* num_attrs, const int32_t* bitdepths,
                                         int32_t* const* values_out,
                                         int8_t* const* lcp_coeffs_out);
int pccb200_attr_lift_decode_multi_batch(int32_t num_units, const pccb200_lod_params* const* lods,
                                         int32_t num_sets, const pccb200_qpset* const* qpsets,
                                         const int32_t* lcp_enabled, const int32_t* const* xyz,
                                         const int32_t* n, int32_t* const* attrs_out,
                                         const int32_t* num_attrs, const int32_t* bitdepths,
                                         const int32_t* const* values_in,
                                         const int8_t* const* lcp_coeffs);
int pccb200_attr_lift_encode_multi_batch_dev(int32_t num_units,
                                             const pccb200_lod_params* const* lods,
                                             int32_t num_sets, const pccb200_qpset* const* qpsets,
                                             const int32_t* lcp_enabled,
                                             const int32_t* const* d_xyz, const int32_t* n,
                                             int32_t* const* d_attrs_inout,
                                             const int32_t* num_attrs, const int32_t* bitdepths,
                                             int32_t* const* d_values_out,
                                             int8_t* const* lcp_coeffs_out);
int pccb200_attr_lift_decode_multi_batch_dev(int32_t num_units,
                                             const pccb200_lod_params* const* lods,
                                             int32_t num_sets, const pccb200_qpset* const* qpsets,
                                             const int32_t* lcp_enabled,
                                             const int32_t* const* d_xyz, const int32_t* n,
                                             int32_t* const* d_attrs_out,
                                             const int32_t* num_attrs, const int32_t* bitdepths,
                                             const int32_t* const* d_values_in,
                                             const int8_t* const* lcp_coeffs);

/* Scalable lifting: the *_multi_batch entries with one pccb200_lod_scalable
 * per unit, scals[u].  The levels of detail are those of
 * pccb200_lod_build_scalable, the quantisation weights those of
 * computeQuantizationWeightsScalable: the encoder's (n, 0)
 * (tmc3/AttributeEncoder.cpp:1390-1395; the encoder codes whole slices, so
 * scals[u] must have min_geom_node_size_log2 == 0 and geom_num_points 0 or
 * n[u]), the decoder's (geom_num_points, min_geom_node_size_log2)
 * (tmc3/AttributeDecoder.cpp:692-697).  lcp rows: 21 entries used (the
 * scalable maxNumDetailLevels).  lod_decimation_type != 0, max_neigh_range < 1
 * and geom_num_points in (0, n[u]) return PCCB200_ERR_INVALID_ARG before a
 * device is looked up.  Workspace: as the *_multi entries, plus 4 bytes per
 * point for the refinement lists and about 1 byte per point of bounding boxes
 * for each neighbour search the concatenation of layers repeats (an estimate,
 * not measured). */
int pccb200_attr_lift_encode_scalable(int32_t num_units, const pccb200_lod_params* const* lods,
                                      const pccb200_lod_scalable* scals, int32_t num_sets,
                                      const pccb200_qpset* const* qpsets,
                                      const int32_t* lcp_enabled, const int32_t* const* xyz,
                                      const int32_t* n, int32_t* const* attrs_inout,
                                      const int32_t* num_attrs, const int32_t* bitdepths,
                                      int32_t* const* values_out, int8_t* const* lcp_coeffs_out);
int pccb200_attr_lift_decode_scalable(int32_t num_units, const pccb200_lod_params* const* lods,
                                      const pccb200_lod_scalable* scals, int32_t num_sets,
                                      const pccb200_qpset* const* qpsets,
                                      const int32_t* lcp_enabled, const int32_t* const* xyz,
                                      const int32_t* n, int32_t* const* attrs_out,
                                      const int32_t* num_attrs, const int32_t* bitdepths,
                                      const int32_t* const* values_in,
                                      const int8_t* const* lcp_coeffs);
int pccb200_attr_lift_encode_scalable_dev(int32_t num_units,
                                          const pccb200_lod_params* const* lods,
                                          const pccb200_lod_scalable* scals, int32_t num_sets,
                                          const pccb200_qpset* const* qpsets,
                                          const int32_t* lcp_enabled,
                                          const int32_t* const* d_xyz, const int32_t* n,
                                          int32_t* const* d_attrs_inout,
                                          const int32_t* num_attrs, const int32_t* bitdepths,
                                          int32_t* const* d_values_out,
                                          int8_t* const* lcp_coeffs_out);
int pccb200_attr_lift_decode_scalable_dev(int32_t num_units,
                                          const pccb200_lod_params* const* lods,
                                          const pccb200_lod_scalable* scals, int32_t num_sets,
                                          const pccb200_qpset* const* qpsets,
                                          const int32_t* lcp_enabled,
                                          const int32_t* const* d_xyz, const int32_t* n,
                                          int32_t* const* d_attrs_out,
                                          const int32_t* num_attrs, const int32_t* bitdepths,
                                          const int32_t* const* d_values_in,
                                          const int8_t* const* lcp_coeffs);

/* ---------------------------------------------------------------------------
 * Spherical coordinates for attribute coding of LiDAR slices (the step before
 * the attribute transforms when attr_aps.spherical_coord_flag is set). */

/* convertXyzToRpl (tmc3/coordinate_conversion.cpp:44-69, with findLaser
 * tmc3/geometry_octree.cpp:855-874 and iatan2 tmc3/misc.cpp:278-309).
 * xyz: N x 3; laser_theta: num_theta elevation tangents (gps.angularTheta);
 * rpl_out: N x 3 (radius, azimuth, laser index); bbox_out: min[3], max[3] of
 * rpl_out (the Box3<int> the reference returns). */
int pccb200_xyz_to_rpl(const int32_t laser_origin[3], const int32_t* laser_theta,
                       int32_t num_theta, const int32_t* xyz, int64_t n,
                       int32_t* rpl_out, int32_t bbox_out[6]);

/* offsetAndScale (tmc3/coordinate_conversion.cpp:108-117), in place. */
int pccb200_offset_and_scale(const int32_t min_pos[3], const int32_t axis_weight[3],
                             int32_t* pos_inout, int64_t n);

/* Both in one call, positions staying on the device in between: what the
 * encoder and decoder do per slice (tmc3/encoder.cpp:1178-1196,
 * tmc3/decoder.cpp:899-918).  min_pos == NULL: offset by the bounding-box
 * minimum of the conversion (the intra case). */
int pccb200_attr_spherical_positions(const int32_t laser_origin[3],
                                     const int32_t* laser_theta, int32_t num_theta,
                                     const int32_t axis_weight[3], const int32_t* min_pos,
                                     const int32_t* xyz, int64_t n, int32_t* pos_out,
                                     int32_t bbox_out[6]);

/* ---------------------------------------------------------------------------
 * Symbol preparation for the entropy coder: the walk over the coefficients
 * right after the forward transform (tmc3/AttributeEncoder.cpp:1279-1291 one
 * component, :1346-1362 three).  For every position with a non-zero
 * coefficient, in coding order:
 *   zero_runs_out[s]       all-zero positions since the previous symbol (the
 *                          argument of PCCResidualsEncoder::encodeRunLength)
 *   values_out[s*A + k]    the coefficients (arguments of encode())
 *   ctx_out[s]             A == 3, may be NULL: b0 | b1<<1 | b2<<2 | b3<<3, the
 *                          context selectors encode() derives from |v1|, |v2|
 *                          (tmc3/AttributeEncoder.cpp:271-296)
 * *count_out symbols; *tail_run_out = all-zero positions after the last one
 * (a final encodeRunLength if non-zero).  Output buffers hold n symbols.
 * coeffs: A x n planar, as written by pccb200_raht_forward. */
int pccb200_coeff_symbols(const int32_t* coeffs, int32_t num_attrs, int32_t n,
                          int32_t* zero_runs_out, int32_t* values_out,
                          uint8_t* ctx_out, int32_t* count_out,
                          int32_t* tail_run_out);

/* pccb200_attr_raht_encode followed by pccb200_coeff_symbols with the
 * coefficients never leaving the device: what crosses PCIe is the symbol
 * stream (usually a small fraction of N x A) and the reconstruction. */
int pccb200_attr_raht_encode_symbols(const pccb200_raht_params* params,
                                     const pccb200_qpset* qpset,
                                     const int32_t* point_qp_offsets,
                                     const int32_t* xyz, int32_t* attrs_inout,
                                     int32_t num_attrs, int32_t n, int32_t bitdepth,
                                     int32_t* zero_runs_out, int32_t* values_out,
                                     uint8_t* ctx_out, int32_t* count_out,
                                     int32_t* tail_run_out);

/* estimateDist2 (tmc3/AttributeEncoder.cpp:1683-1720; per slice from
 * tmc3/encoder.cpp:1199-1206: abh.attr_dist2_delta = result - aps.dist2).
 * xyz: N x 3 in coding order.  *shift_bits_out = the reference's return value. */
int pccb200_estimate_dist2(const int32_t* xyz, int32_t n, int32_t sampling_period,
                           int32_t search_range, float percentile_estimate,
                           int32_t* shift_bits_out);

/* Predicting transform decoder (attr_encoding 0, transformType 1) -------------
 *
 * AttributeDecoder::decode{Colors,Reflectances}Pred
 * (tmc3/AttributeDecoder.cpp:328-391,446-523) after its entropy decoding:
 * values_in holds, per point in coding (predictor) order, the values the
 * reference's loop decodes (zero runs expanded: decodeRunLength / decode),
 * with the prediction mode still in their low bits.  The library applies the
 * rest of the loop: fixed-weight quantisation weights (quant_neigh_weight),
 * the quantisers of the point's level (quantLayer) and qp offsets, the mode's
 * eligibility from the neighbours' reconstructed values against
 * adaptive_prediction_threshold << max(0, bitdepth - 8), the mode unpacked
 * from the values, the prediction, dequantisation, inter-component prediction
 * and the clip to [0, 2^bitdepth - 1].  The output is the decoded attribute
 * per point, in point order, bit-identical to the reference's.
 *
 * A point's prediction reads the reconstructions of its neighbours, whose
 * predictor indexes must be below its own (the levels of detail of the
 * predicting transform have that form, also with intra-LoD prediction).
 * Predictors that break it return PCCB200_ERR_INVALID_ARG before any decoding
 * starts.  Scalable lifting handles and inter-frame prediction are not
 * supported (PCCB200_ERR_UNSUPPORTED for a scalable handle).
 *
 * qpset: fixed_point_qp_offset 0, as deriveQpSet sets it for this transform.
 * point_qp_offsets: N x 2 in point order (the region offsets of
 * QpSet::quantizers), or NULL.  icp_coeffs: a host row of PCCB200_MAX_LODS
 * triplets, abh.icpCoeffs per level of detail, or NULL when the brick header
 * carries none (icpPresent false). */
typedef struct pccb200_pred_params {
  int32_t max_num_direct_predictors;      /* 0..3 */
  int32_t direct_avg_predictor_disabled;  /* direct_avg_predictor_disabled_flag */
  int32_t adaptive_prediction_threshold;  /* unscaled, as in the APS */
  int32_t icp_enabled;                    /* inter_component_prediction_enabled_flag */
} pccb200_pred_params;

#define PCCB200_MAX_PRED_SETS 4

/* On a pccb200_lod_create / pccb200_lod_import handle: one attribute of
 * num_attrs (1 or 3) components.  values_in, attrs_out: N x num_attrs. */
int pccb200_attr_pred_decode_lod(pccb200_lod_handle handle, const pccb200_qpset* qpset,
                                 const pccb200_pred_params* pred,
                                 const int32_t quant_neigh_weight[3],
                                 const int32_t* point_qp_offsets, const int8_t* icp_coeffs,
                                 const int32_t* values_in, int32_t num_attrs, int32_t bitdepth,
                                 int32_t* attrs_out);

/* num_units units (slices or frames), each with its own LoD parameters
 * lods[u] (pred_weight_blending and the intra-LoD settings included),
 * positions xyz[u] (n[u] x 3), quant_neigh_weight[3u..3u+2] and qp offsets
 * point_qp_offsets[u] (or point_qp_offsets NULL, or an entry NULL), and
 * num_sets (1..PCCB200_MAX_PRED_SETS) attribute sets sharing its levels of
 * detail.  qpsets[s], pred[s], num_attrs[s], bitdepths[s] are per set;
 * values_in[u * num_sets + s], icp_coeffs[u * num_sets + s] (or icp_coeffs
 * NULL, or an entry NULL) and attrs_out[u * num_sets + s] per unit and set.
 * Units are spread over the library's lanes; the units of a lane decode in one
 * dataflow launch.  Results are bit-identical to one call per unit.
 * The _dev entry takes device pointers for xyz, point_qp_offsets, values_in and
 * attrs_out; everything else stays on the host. */
int pccb200_attr_pred_decode_multi_batch(
  int32_t num_units, const pccb200_lod_params* const* lods, const int32_t* quant_neigh_weight,
  int32_t num_sets, const pccb200_qpset* const* qpsets, const pccb200_pred_params* pred,
  const int32_t* num_attrs, const int32_t* bitdepths, const int32_t* const* xyz, const int32_t* n,
  const int32_t* const* point_qp_offsets, const int32_t* const* values_in,
  const int8_t* const* icp_coeffs, int32_t* const* attrs_out);
int pccb200_attr_pred_decode_multi_batch_dev(
  int32_t num_units, const pccb200_lod_params* const* lods, const int32_t* quant_neigh_weight,
  int32_t num_sets, const pccb200_qpset* const* qpsets, const pccb200_pred_params* pred,
  const int32_t* num_attrs, const int32_t* bitdepths, const int32_t* const* d_xyz,
  const int32_t* n, const int32_t* const* d_point_qp_offsets, const int32_t* const* d_values_in,
  const int8_t* const* icp_coeffs, int32_t* const* d_attrs_out);

#ifdef __cplusplus
}
#endif
#endif /* PCC_ATTR_B200_H */
