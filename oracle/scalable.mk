# oracle/scalable.mk — TEST INFRASTRUCTURE ONLY.
#
#  make -f scalable.mk scalableref : the reference's scalable-lifting LoD build,
#      lifting encoder and decoder (ref_shim_scalable_enc.cpp /
#      ref_shim_scalable_dec.cpp, which #include tmc3/AttributeEncoder.cpp and
#      tmc3/AttributeDecoder.cpp from where they lie), linked with the
#      position-independent reference objects of `make liftref`, into
#      _ref/libtmc13_scalable.so.  Needs the reference tree.
include Makefile

scalableref: _ref/libtmc13_scalable.so
SCALABLE_SHIMS = ref_shim_scalable_enc.cpp ref_shim_scalable_dec.cpp
_ref/libtmc13_scalable.so: $(SCALABLE_SHIMS) $(LIFT_OBJS) ../include/pcc_attr_b200.h
	$(CXX) -std=c++14 $(OPT) -fPIC -shared -w $(CODEC_INC) $(SCALABLE_SHIMS) $(LIFT_OBJS) -o $@
