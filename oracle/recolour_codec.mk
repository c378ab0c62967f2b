# oracle/recolour_codec.mk — TEST INFRASTRUCTURE ONLY.
#
#  make -f recolour_codec.mk kdtreeref : the reference's nanoflann kd-tree
#      (dependencies/nanoflann, unmodified, through the adaptor the reference
#      recolours with) and the compiled std::sort behind ref_shim_kdtree.cpp,
#      into _ref/libtmc13_kdtree.so.
#  make -f recolour_codec.mk recolourcodec : the reference's tmc3 with
#      pcc::recolour replaced by the product's drop-in translation unit
#      (mpeg-pcc-tmc13_b200/host/recolour_dropin.cpp) and linked against
#      libpcc_attr_b200.so (_ref/tmc3_b200_recolour).  The reference's own
#      recolour stays in the binary under the name pccb200_reference_recolour
#      (objcopy --redefine-sym on pointset_processing.o), as the drop-in's
#      fallback.  Everything else is the objects of `make codec`; _ref/tmc3_ref
#      and _ref/tmc3_b200 are untouched.
#  Both need the reference tree.
include Makefile

kdtreeref: _ref/libtmc13_kdtree.so
_ref/libtmc13_kdtree.so: ref_shim_kdtree.cpp
	@test -d $(REF)/tmc3 || { echo "reference tree $(REF) not present: keeping prebuilt _ref"; exit 0; }
	mkdir -p _ref/gen
	printf '#pragma once\n#define HAVE_GETRUSAGE 1\n' > _ref/gen/TMC3Config.h
	$(CXX) -std=c++14 $(OPT) -fPIC -shared -w $(REF_INC) ref_shim_kdtree.cpp -o $@

recolourcodec: _ref/tmc3_b200_recolour

RECOLOUR_FN = _ZN3pcc8recolourERKNS_20AttributeDescriptionERKNS_14RecolourParamsERKNS_12PCCPointSet3EfNS_4Vec3IiEEPS6_
_ref/obj/pointset_processing_b200.o: _ref/obj/pointset_processing.o
	objcopy --redefine-sym $(RECOLOUR_FN)=pccb200_reference_recolour $< $@
_ref/obj/recolour_dropin.o: $(PKG)/host/recolour_dropin.cpp ../include/pcc_attr_b200.h _ref/gen/version.cpp
	$(CXX) -std=c++14 $(OPT) -w $(CODEC_INC) -c $< -o $@

RECOLOUR_B200_OBJS = $(filter-out _ref/obj/pointset_processing.o,$(CODEC_OBJS)) _ref/obj/RAHT.o \
  _ref/obj/pointset_processing_b200.o _ref/obj/recolour_dropin.o
_ref/tmc3_b200_recolour: $(RECOLOUR_B200_OBJS)
	$(CXX) $^ -L$(PKG) -lpcc_attr_b200 -Wl,-rpath,'$$ORIGIN/../../mpeg-pcc-tmc13_b200' -o $@
