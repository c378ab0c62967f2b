# oracle/lift_codec.mk — TEST INFRASTRUCTURE ONLY.
#
#  make -f lift_codec.mk liftcodec : the reference's tmc3 with the four lifting
#      coding bodies (AttributeEncoder::encode{Colors,Reflectances}Lift,
#      AttributeDecoder::decode{Colors,Reflectances}Lift) replaced by the
#      product's drop-in translation unit (mpeg-pcc-tmc13_b200/host/
#      lift_dropin.cpp) and linked against libpcc_attr_b200.so
#      (_ref/tmc3_b200_lift).  Everything else is the objects of _ref/tmc3_b200
#      (RAHT and LoD drop-ins included); _ref/tmc3_ref and _ref/tmc3_b200 are
#      untouched.  Needs the reference tree.
#
# The bodies are called from encode() / decode() in the same object, so a
# rename of the definition (objcopy --redefine-sym) would rename the calls as
# well.  Instead the copies AttributeEncoder_lift.o / AttributeDecoder_lift.o
# WEAKEN the four definitions, so that the drop-in's strong ones serve the
# calls, and add a global alias pccb200_reference_<name> at the offset of each
# body (the drop-in's fallback) and of each residual-coder method the drop-in's
# entropy loops call.  The offsets are read from the object's symbol table.
include Makefile

liftcodec: _ref/tmc3_b200_lift

ENC_BODIES = \
  encodeColorsLift=_ZN3pcc16AttributeEncoder16encodeColorsLiftERKNS_20AttributeDescriptionERKNS_21AttributeParameterSetERKNS_5QpSetERNS_12PCCPointSet3ERNS_19PCCResidualsEncoderE \
  encodeReflectancesLift=_ZN3pcc16AttributeEncoder22encodeReflectancesLiftERKNS_20AttributeDescriptionERKNS_21AttributeParameterSetERKNS_5QpSetERNS_12PCCPointSet3ERNS_19PCCResidualsEncoderERNS_24AttributeInterPredParamsE
ENC_CODER = \
  encodeRunLength=_ZN3pcc19PCCResidualsEncoder15encodeRunLengthEi \
  encode1=_ZN3pcc19PCCResidualsEncoder6encodeEi \
  encode3=_ZN3pcc19PCCResidualsEncoder6encodeEiii
DEC_BODIES = \
  decodeColorsLift=_ZN3pcc16AttributeDecoder16decodeColorsLiftERKNS_20AttributeDescriptionERKNS_21AttributeParameterSetERKNS_20AttributeBrickHeaderERKNS_5QpSetEiiRNS_19PCCResidualsDecoderERNS_12PCCPointSet3E \
  decodeReflectancesLift=_ZN3pcc16AttributeDecoder22decodeReflectancesLiftERKNS_20AttributeDescriptionERKNS_21AttributeParameterSetERKNS_20AttributeBrickHeaderERKNS_5QpSetEiiRNS_19PCCResidualsDecoderERNS_12PCCPointSet3ERKNS_24AttributeInterPredParamsE
DEC_CODER = \
  decodeRunLength=_ZN3pcc19PCCResidualsDecoder15decodeRunLengthEv \
  decode3=_ZN3pcc19PCCResidualsDecoder6decodeEPi \
  decode1=_ZN3pcc19PCCResidualsDecoder6decodeEv

# $(call weaken_alias,<bodies>,<coder methods>): objcopy $< -> $@ with every body
# weakened and every body and method aliased as pccb200_reference_<name>
define weaken_alias
	flags=""; for p in $(1) $(2); do \
	  a=$${p%%=*}; s=$${p#*=}; \
	  loc=$$(objdump -t $< | awk -v s=$$s '$$NF == s && $$(NF-2) ~ /^\.text/ { print $$(NF-2) ":0x" $$1 }'); \
	  test -n "$$loc" || { echo "$$s not defined in $<"; exit 1; }; \
	  flags="$$flags --add-symbol pccb200_reference_$$a=$$loc,global,function"; \
	done; \
	for p in $(1); do flags="$$flags --weaken-symbol=$${p#*=}"; done; \
	objcopy $$flags $< $@
endef

_ref/obj/AttributeEncoder_lift.o: _ref/obj/AttributeEncoder.o lift_codec.mk
	$(call weaken_alias,$(ENC_BODIES),$(ENC_CODER))
_ref/obj/AttributeDecoder_lift.o: _ref/obj/AttributeDecoder.o lift_codec.mk
	$(call weaken_alias,$(DEC_BODIES),$(DEC_CODER))
_ref/obj/lift_dropin.o: $(PKG)/host/lift_dropin.cpp $(PKG)/host/qpset_flatten.h \
  ../include/pcc_attr_b200.h _ref/gen/version.cpp
	$(CXX) -std=c++14 $(OPT) -w $(CODEC_INC) -c $< -o $@

LIFT_B200_OBJS = $(filter-out _ref/obj/AttributeEncoder.o _ref/obj/AttributeDecoder.o,$(B200_OBJS)) \
  _ref/obj/AttributeEncoder_lift.o _ref/obj/AttributeDecoder_lift.o _ref/obj/lift_dropin.o
_ref/tmc3_b200_lift: $(LIFT_B200_OBJS)
	$(CXX) $^ -L$(PKG) -lpcc_attr_b200 -Wl,-rpath,'$$ORIGIN/../../mpeg-pcc-tmc13_b200' -o $@
