// lift_dropin.cpp — host-side mirror of the reference interface for the
// lifting transform's coding loops: a translation unit that DEFINES the
// reference's own member functions
//
//   pcc::AttributeEncoder::encodeColorsLift        (tmc3/AttributeEncoder.cpp:1379-1494)
//   pcc::AttributeEncoder::encodeReflectancesLift  (tmc3/AttributeEncoder.cpp:1543-1648)
//   pcc::AttributeDecoder::decodeColorsLift        (tmc3/AttributeDecoder.cpp:678-770)
//   pcc::AttributeDecoder::decodeReflectancesLift  (tmc3/AttributeDecoder.cpp:774-857)
//
// with their exact C++ signatures.  The levels of detail the caller built
// (_lods, whoever made them: the reference or lod_dropin.cpp) are handed to the
// library with pccb200_lod_import, and pccb200_attr_lift_encode_lod /
// _decode_lod run quantisation weights, forward lifting, last-component
// prediction, quantisation, inverse lifting and the clip on the device.  The
// entropy coding stays the reference's: the encoder runs its zero-run / encode
// loop over the returned values in coding order (and stores the LCP
// coefficients in the brick header), the decoder runs its decode loop first and
// hands the values to one library call.  Reconstructions come back clipped in
// point order.  The callers AttributeEncoder::encode and AttributeDecoder::decode
// are unchanged, and the bitstream stays byte-identical
// (tests/test_lift_dropin.py::test_whole_codec_lift).
//
// The four bodies and the residual coder sit in the same object files as their
// callers, so a rename of the definition would rename the calls too.
// oracle/lift_codec.mk instead WEAKENS the four definitions in
// AttributeEncoder.o / AttributeDecoder.o (this unit's strong ones win at link
// time) and adds an alias for each of them and for the six residual-coder
// methods the loops call (objcopy --add-symbol at the definition's offset).
// The aliased bodies are the fallback for what the library does not take:
// inter-frame prediction (enableAttrInterPred, attrInterIntraSliceRDO), more
// than PCCB200_MAX_LODS levels of detail or qp layers, predictors outside the
// library's form, and predictors that reference their own level of detail.
// With PCCB200_DROPIN_STRICT=1 in the environment those throw instead, so
// that a run proves the library did the work.  Any other library error throws
// std::runtime_error.  A maintainer would instead rename the bodies in
// AttributeEncoder.cpp / AttributeDecoder.cpp and call the residual coder
// directly; see INTEGRATION.md.
#include <cstdlib>
#include <stdexcept>
#include <string>
#include <vector>

#include "AttributeDecoder.h"
#include "AttributeEncoder.h"

#include "pcc_attr_b200.h"
#include "qpset_flatten.h"

namespace pcc {

// The reference's own definitions under their link-time names (Itanium C++
// ABI: a member function takes `this` as its first argument).
extern "C" void pccb200_reference_encodeColorsLift(
  AttributeEncoder* self, const AttributeDescription& desc, const AttributeParameterSet& aps,
  const QpSet& qpSet, PCCPointSet3& pointCloud, PCCResidualsEncoder& encoder);
extern "C" void pccb200_reference_encodeReflectancesLift(
  AttributeEncoder* self, const AttributeDescription& desc, const AttributeParameterSet& aps,
  const QpSet& qpSet, PCCPointSet3& pointCloud, PCCResidualsEncoder& encoder,
  AttributeInterPredParams& attrInterPredParams);
extern "C" void pccb200_reference_decodeColorsLift(
  AttributeDecoder* self, const AttributeDescription& desc, const AttributeParameterSet& aps,
  const AttributeBrickHeader& abh, const QpSet& qpSet, int geom_num_points_minus1,
  int minGeomNodeSizeLog2, PCCResidualsDecoder& decoder, PCCPointSet3& pointCloud);
extern "C" void pccb200_reference_decodeReflectancesLift(
  AttributeDecoder* self, const AttributeDescription& desc, const AttributeParameterSet& aps,
  const AttributeBrickHeader& abh, const QpSet& qpSet, int geom_num_points_minus1,
  int minGeomNodeSizeLog2, PCCResidualsDecoder& decoder, PCCPointSet3& pointCloud,
  const AttributeInterPredParams& attrInterPredParams);

// PCCResidualsEncoder::encodeRunLength(int), ::encode(int32_t),
// ::encode(int32_t, int32_t, int32_t)
extern "C" void pccb200_reference_encodeRunLength(PCCResidualsEncoder* self, int runLength);
extern "C" void pccb200_reference_encode1(PCCResidualsEncoder* self, int32_t value);
extern "C" void pccb200_reference_encode3(
  PCCResidualsEncoder* self, int32_t value0, int32_t value1, int32_t value2);
// PCCResidualsDecoder::decodeRunLength(), ::decode(int32_t[3]), ::decode()
extern "C" int pccb200_reference_decodeRunLength(PCCResidualsDecoder* self);
extern "C" void pccb200_reference_decode3(PCCResidualsDecoder* self, int32_t values[3]);
extern "C" int32_t pccb200_reference_decode1(PCCResidualsDecoder* self);

namespace {

bool
strict()
{
  const char* s = std::getenv("PCCB200_DROPIN_STRICT");
  return s && s[0] == '1';
}

// true: the reference body does the work (or, strict, a throw)
bool
fall_back(const char* why)
{
  if (strict())
    throw std::runtime_error(std::string("lift drop-in: ") + why);
  return true;
}

void
check(int rc, const char* what)
{
  if (rc != PCCB200_OK)
    throw std::runtime_error(
      std::string("lift drop-in: ") + what + ": " + pccb200_last_error());
}

// The levels of detail in the library's form, or false when they are outside
// it (more levels than PCCB200_MAX_LODS, more than three neighbours, a weight
// of 2^32 or more) or reference their own level of detail (the lifting passes
// need strictly coarser neighbours; the decoder must know before it reads its
// stream, since the reference body would then read the same symbols).
bool
flatten_lods(const AttributeLods& lods, std::vector<pccb200_predictor>& preds)
{
  const size_t n = lods.predictors.size();
  const size_t levels = lods.numPointsInLod.size();
  if (n == 0 || n >= (size_t(1) << 31) || levels == 0 || levels > PCCB200_MAX_LODS
      || lods.indexes.size() != n)
    return false;
  preds.resize(n);
  size_t lod = 0;
  for (size_t i = 0; i < n; i++) {
    while (lod < levels && i >= lods.numPointsInLod[lod])
      lod++;
    const size_t start = lod ? lods.numPointsInLod[lod - 1] : 0;
    const PCCPredictor& p = lods.predictors[i];
    if (p.neighborCount > 3)
      return false;
    pccb200_predictor& q = preds[i];
    q = pccb200_predictor{};
    q.neighbor_count = p.neighborCount;
    for (uint32_t j = 0; j < p.neighborCount; j++) {
      const PCCNeighborInfo& nb = p.neighbors[j];
      if (nb.weight >> 32 || (lod && nb.predictorIndex >= start))
        return false;
      q.predictor_index[j] = nb.predictorIndex;
      q.weight[j] = uint32_t(nb.weight);
    }
  }
  return true;
}

// owns a pccb200_lod_handle
struct Handle {
  pccb200_lod_handle h = nullptr;
  ~Handle() { pccb200_lod_destroy(h); }
};

// imports lods; scal: scalable lifting's (geom_num_points, minGeomNodeSizeLog2)
// weights, or null
void
import_lods(const AttributeLods& lods, const std::vector<pccb200_predictor>& preds,
            int numDetailLevels, const pccb200_lod_scalable* scal, Handle& out)
{
  check(pccb200_lod_import(preds.data(), lods.indexes.data(), int32_t(preds.size()),
                           lods.numPointsInLod.data(), int32_t(lods.numPointsInLod.size()),
                           numDetailLevels, scal, &out.h),
        "pccb200_lod_import failed");
}

// QpSet::regionQpOffset per point (point order), or an empty vector when no
// region applies
std::vector<int32_t>
region_qp_offsets(const QpSet& qpSet, const PCCPointSet3& cloud)
{
  std::vector<int32_t> qpo;
  if (qpSet.regions.empty())
    return qpo;
  const size_t n = cloud.getPointCount();
  qpo.resize(2 * n);
  for (size_t i = 0; i < n; i++) {
    const Qps o = qpSet.regionQpOffset(cloud[i]);
    qpo[2 * i] = o[0];
    qpo[2 * i + 1] = o[1];
  }
  return qpo;
}

pccb200_lod_scalable
scalable_weights(int64_t geomNumPoints, int minGeomNodeSizeLog2)
{
  pccb200_lod_scalable s = {};
  s.max_neigh_range = 1;  // (not read by pccb200_lod_import)
  s.min_geom_node_size_log2 = minGeomNodeSizeLog2;
  s.geom_num_points = geomNumPoints;
  return s;
}

}  // namespace

//============================================================================
// encoder

void
AttributeEncoder::encodeColorsLift(
  const AttributeDescription& desc,
  const AttributeParameterSet& aps,
  const QpSet& qpSet,
  PCCPointSet3& pointCloud,
  PCCResidualsEncoder& encoder)
{
  const size_t n = pointCloud.getPointCount();
  std::vector<pccb200_predictor> preds;
  pccb200_qpset q;
  if (n != _lods.predictors.size() || !flatten_lods(_lods, preds) || !qpset_fits(qpSet)
      || aps.maxNumDetailLevels() > PCCB200_MAX_LODS) {
    if (fall_back("levels of detail or qp layers outside the library's range"))
      return pccb200_reference_encodeColorsLift(this, desc, aps, qpSet, pointCloud, encoder);
  }
  const pccb200_lod_scalable scal = scalable_weights(int64_t(n), 0);
  flatten_qpset(qpSet, q);
  Handle h;
  import_lods(_lods, preds, aps.maxNumDetailLevels(),
              aps.scalable_lifting_enabled_flag ? &scal : nullptr, h);

  std::vector<int32_t> attrs(3 * n), values(3 * n);
  for (size_t i = 0; i < n; i++) {
    const Vec3<attr_t> c = pointCloud.getColor(i);
    for (int k = 0; k < 3; k++)
      attrs[3 * i + k] = c[k];
  }
  const std::vector<int32_t> qpo = region_qp_offsets(qpSet, pointCloud);
  const bool lcp = aps.last_component_prediction_enabled_flag;
  int8_t lcpRow[PCCB200_MAX_LODS] = {};
  const int rc = pccb200_attr_lift_encode_lod(
    h.h, &q, lcp, qpo.empty() ? nullptr : qpo.data(), attrs.data(), 3, desc.bitdepth,
    values.data(), lcpRow);
  if (rc == PCCB200_ERR_UNSUPPORTED
      && fall_back("a predictor references its own level of detail"))
    return pccb200_reference_encodeColorsLift(this, desc, aps, qpSet, pointCloud, encoder);
  check(rc, "pccb200_attr_lift_encode_lod failed");

  if (lcp)
    _abh->attrLcpCoeffs.assign(lcpRow, lcpRow + aps.maxNumDetailLevels());

  int zeroRun = 0;
  for (size_t i = 0; i < n; i++) {
    const int32_t* v = &values[3 * i];
    if (!v[0] && !v[1] && !v[2])
      ++zeroRun;
    else {
      pccb200_reference_encodeRunLength(&encoder, zeroRun);
      pccb200_reference_encode3(&encoder, v[0], v[1], v[2]);
      zeroRun = 0;
    }
  }
  if (zeroRun)
    pccb200_reference_encodeRunLength(&encoder, zeroRun);

  for (size_t i = 0; i < n; i++)
    pointCloud.setColor(
      i, Vec3<attr_t>(attr_t(attrs[3 * i]), attr_t(attrs[3 * i + 1]), attr_t(attrs[3 * i + 2])));
}

void
AttributeEncoder::encodeReflectancesLift(
  const AttributeDescription& desc,
  const AttributeParameterSet& aps,
  const QpSet& qpSet,
  PCCPointSet3& pointCloud,
  PCCResidualsEncoder& encoder,
  AttributeInterPredParams& attrInterPredParams)
{
  const size_t n = pointCloud.getPointCount();
  std::vector<pccb200_predictor> preds;
  pccb200_qpset q;
  const char* why = nullptr;
  if (attrInterPredParams.enableAttrInterPred || attrInterPredParams.attrInterIntraSliceRDO)
    why = "inter-frame prediction";
  else if (n != _lods.predictors.size() || !flatten_lods(_lods, preds) || !qpset_fits(qpSet)
           || aps.maxNumDetailLevels() > PCCB200_MAX_LODS)
    why = "levels of detail or qp layers outside the library's range";
  if (why && fall_back(why))
    return pccb200_reference_encodeReflectancesLift(
      this, desc, aps, qpSet, pointCloud, encoder, attrInterPredParams);
  attrInterPredParams.distEstimate = 0.;
  const pccb200_lod_scalable scal = scalable_weights(int64_t(n), 0);
  flatten_qpset(qpSet, q);
  Handle h;
  import_lods(_lods, preds, aps.maxNumDetailLevels(),
              aps.scalable_lifting_enabled_flag ? &scal : nullptr, h);

  std::vector<int32_t> attrs(n), values(n);
  for (size_t i = 0; i < n; i++)
    attrs[i] = pointCloud.getReflectance(i);
  const std::vector<int32_t> qpo = region_qp_offsets(qpSet, pointCloud);
  const int rc = pccb200_attr_lift_encode_lod(
    h.h, &q, 0, qpo.empty() ? nullptr : qpo.data(), attrs.data(), 1, desc.bitdepth,
    values.data(), nullptr);
  if (rc == PCCB200_ERR_UNSUPPORTED
      && fall_back("a predictor references its own level of detail"))
    return pccb200_reference_encodeReflectancesLift(
      this, desc, aps, qpSet, pointCloud, encoder, attrInterPredParams);
  check(rc, "pccb200_attr_lift_encode_lod failed");

  int zeroRun = 0;
  for (size_t i = 0; i < n; i++) {
    if (!values[i])
      ++zeroRun;
    else {
      pccb200_reference_encodeRunLength(&encoder, zeroRun);
      pccb200_reference_encode1(&encoder, values[i]);
      zeroRun = 0;
    }
  }
  if (zeroRun)
    pccb200_reference_encodeRunLength(&encoder, zeroRun);

  for (size_t i = 0; i < n; i++)
    pointCloud.setReflectance(i, attr_t(attrs[i]));
}

//============================================================================
// decoder

void
AttributeDecoder::decodeColorsLift(
  const AttributeDescription& desc,
  const AttributeParameterSet& aps,
  const AttributeBrickHeader& abh,
  const QpSet& qpSet,
  int geom_num_points_minus1,
  int minGeomNodeSizeLog2,
  PCCResidualsDecoder& decoder,
  PCCPointSet3& pointCloud)
{
  const size_t n = pointCloud.getPointCount();
  std::vector<pccb200_predictor> preds;
  pccb200_qpset q;
  const bool lcp = aps.last_component_prediction_enabled_flag;
  if (n != _lods.predictors.size() || !flatten_lods(_lods, preds) || !qpset_fits(qpSet)
      || aps.maxNumDetailLevels() > PCCB200_MAX_LODS
      || (lcp && int(abh.attrLcpCoeffs.size()) < int(_lods.numPointsInLod.size()))) {
    if (fall_back("levels of detail or qp layers outside the library's range"))
      return pccb200_reference_decodeColorsLift(
        this, desc, aps, abh, qpSet, geom_num_points_minus1, minGeomNodeSizeLog2, decoder,
        pointCloud);
  }

  // the reference's decode loop, values in coding order
  std::vector<int32_t> values(3 * n);
  int zeroRunRem = 0;
  for (size_t i = 0; i < n; i++) {
    if (--zeroRunRem < 0)
      zeroRunRem = pccb200_reference_decodeRunLength(&decoder);
    if (!zeroRunRem)
      pccb200_reference_decode3(&decoder, &values[3 * i]);
  }

  const pccb200_lod_scalable scal =
    scalable_weights(int64_t(geom_num_points_minus1) + 1, minGeomNodeSizeLog2);
  flatten_qpset(qpSet, q);
  Handle h;
  import_lods(_lods, preds, aps.maxNumDetailLevels(),
              aps.scalable_lifting_enabled_flag ? &scal : nullptr, h);
  int8_t lcpRow[PCCB200_MAX_LODS] = {};
  for (int l = 0; lcp && l < int(abh.attrLcpCoeffs.size()) && l < PCCB200_MAX_LODS; l++)
    lcpRow[l] = abh.attrLcpCoeffs[l];
  const std::vector<int32_t> qpo = region_qp_offsets(qpSet, pointCloud);
  std::vector<int32_t> attrs(3 * n);
  check(pccb200_attr_lift_decode_lod(h.h, &q, lcp, qpo.empty() ? nullptr : qpo.data(),
                                     attrs.data(), 3, desc.bitdepth, values.data(),
                                     lcp ? lcpRow : nullptr),
        "pccb200_attr_lift_decode_lod failed");

  for (size_t i = 0; i < n; i++)
    pointCloud.setColor(
      i, Vec3<attr_t>(attr_t(attrs[3 * i]), attr_t(attrs[3 * i + 1]), attr_t(attrs[3 * i + 2])));
}

void
AttributeDecoder::decodeReflectancesLift(
  const AttributeDescription& desc,
  const AttributeParameterSet& aps,
  const AttributeBrickHeader& abh,
  const QpSet& qpSet,
  int geom_num_points_minus1,
  int minGeomNodeSizeLog2,
  PCCResidualsDecoder& decoder,
  PCCPointSet3& pointCloud,
  const AttributeInterPredParams& attrInterPredParams)
{
  const size_t n = pointCloud.getPointCount();
  std::vector<pccb200_predictor> preds;
  pccb200_qpset q;
  const char* why = nullptr;
  if (attrInterPredParams.enableAttrInterPred || attrInterPredParams.attrInterIntraSliceRDO)
    why = "inter-frame prediction";
  else if (n != _lods.predictors.size() || !flatten_lods(_lods, preds) || !qpset_fits(qpSet)
           || aps.maxNumDetailLevels() > PCCB200_MAX_LODS)
    why = "levels of detail or qp layers outside the library's range";
  if (why && fall_back(why))
    return pccb200_reference_decodeReflectancesLift(
      this, desc, aps, abh, qpSet, geom_num_points_minus1, minGeomNodeSizeLog2, decoder,
      pointCloud, attrInterPredParams);

  std::vector<int32_t> values(n);
  int zeroRunRem = 0;
  for (size_t i = 0; i < n; i++) {
    if (--zeroRunRem < 0)
      zeroRunRem = pccb200_reference_decodeRunLength(&decoder);
    if (!zeroRunRem)
      values[i] = pccb200_reference_decode1(&decoder);
  }

  const pccb200_lod_scalable scal =
    scalable_weights(int64_t(geom_num_points_minus1) + 1, minGeomNodeSizeLog2);
  flatten_qpset(qpSet, q);
  Handle h;
  import_lods(_lods, preds, aps.maxNumDetailLevels(),
              aps.scalable_lifting_enabled_flag ? &scal : nullptr, h);
  const std::vector<int32_t> qpo = region_qp_offsets(qpSet, pointCloud);
  std::vector<int32_t> attrs(n);
  check(pccb200_attr_lift_decode_lod(h.h, &q, 0, qpo.empty() ? nullptr : qpo.data(),
                                     attrs.data(), 1, desc.bitdepth, values.data(), nullptr),
        "pccb200_attr_lift_decode_lod failed");

  for (size_t i = 0; i < n; i++)
    pointCloud.setReflectance(i, attr_t(attrs[i]));
}

}  // namespace pcc
