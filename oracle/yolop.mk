# oracle/yolop.mk -- builds, with oracle/Makefile's flags and variables (included below),
#   libyolop_oracle.so            the CPU oracle of the YOLOP pre- and post-process (yolop_oracle.c, on cls_oracle.c's resize)
#   _ref/libref_yolop_host.so     YOLOP's own nms() and get_rect (yolop/common.hpp), compiled where they lie
#   _ref/libref_yolop.so          YOLOP's own YoloLayer plugin kernel (yolop/yololayer.cu)
# `make -f yolop.mk` builds the three (the two reference libraries only where the reference tree is present);
# tensorrtx_b200.build.build_oracle() runs it after oracle/Makefile.
yolop:

include $(dir $(abspath $(lastword $(MAKEFILE_LIST))))Makefile

YOLOP_REF := $(HERE)_ref/libref_yolop_host.so $(HERE)_ref/libref_yolop.so
ifneq ($(wildcard $(REF)),)
yolop: $(HERE)libyolop_oracle.so $(YOLOP_REF)
else
yolop: $(HERE)libyolop_oracle.so
endif

$(HERE)libyolop_oracle.so: $(HERE)yolop_oracle.c $(HERE)cls_oracle.c
	$(CC) $(CFLAGS) -o $@ $< -lm

$(HERE)_ref/libref_yolop_host.so: HOSTEXTRA := -ffp-contract=off
$(HERE)_ref/libref_yolop_host.so: $(HERE)ref_wrap_yolop_host.cpp $(REF)/yolop/common.hpp
	@mkdir -p $(HERE)_ref
	$(CXX) $(HOSTFLAGS) -DTRTX_MOCK_NO_REGISTRAR -I$(REF)/yolop -o $@ $<

$(HERE)_ref/libref_yolop.so: $(HERE)ref_wrap_yolop.cu $(REF)/yolop/yololayer.cu
	@mkdir -p $(HERE)_ref
	$(NVCC) $(NVFLAGS) -I$(REF)/yolop -o $@ $^

.PHONY: yolop
