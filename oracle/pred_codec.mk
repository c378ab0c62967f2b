# oracle/pred_codec.mk — TEST INFRASTRUCTURE ONLY.
#
#  make -f pred_codec.mk predref : the reference's predicting-transform encoder
#      and decoder bodies (ref_shim_predenc.cpp / ref_shim_preddec.cpp, which
#      #include tmc3/AttributeEncoder.cpp and tmc3/AttributeDecoder.cpp from
#      where they lie), linked with the position-independent reference objects
#      of `make liftref`, into _ref/libtmc13_pred.so.  Needs the reference tree.
include Makefile

predref: _ref/libtmc13_pred.so
PRED_SHIMS = ref_shim_predenc.cpp ref_shim_preddec.cpp
_ref/libtmc13_pred.so: $(PRED_SHIMS) $(LIFT_OBJS) ../include/pcc_attr_b200.h
	$(CXX) -std=c++14 $(OPT) -fPIC -shared -w $(CODEC_INC) $(PRED_SHIMS) $(LIFT_OBJS) -o $@
