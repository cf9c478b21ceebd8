# oracle/ufld.mk -- builds, with oracle/Makefile's flags and variables (included below),
#   libufld_oracle.so             the CPU oracle of the UFLD pre- and post-process (ufld_oracle.c, on cls_oracle.c's resize)
#   _ref/libref_ufld_host.so      the driver's own argmax and softmax_mul (ufld/lane_det.cpp), compiled where it lies against
#                                 shim_ufld with its main renamed, only where the reference tree is present.  The driver loop
#                                 sits inside main(), so the oracle restates it.
# tensorrtx_b200.build.build_oracle() runs `make -f ufld.mk` after oracle/Makefile, yolop.mk, detr.mk and centernet.mk.
ufld:

include $(dir $(abspath $(lastword $(MAKEFILE_LIST))))Makefile

ifneq ($(wildcard $(REF)),)
ufld: $(HERE)libufld_oracle.so $(HERE)_ref/libref_ufld_host.so
else
ufld: $(HERE)libufld_oracle.so
endif

$(HERE)libufld_oracle.so: $(HERE)ufld_oracle.c $(HERE)cls_oracle.c
	$(CC) $(CFLAGS) -o $@ $< -lm

# -ffp-contract=off as the oracle; the engine code that nothing exported reaches is dropped with its sections
# (-Wl,--gc-sections), and with it every reference to TensorRT and CUDA entry points this image has no library for.
$(HERE)_ref/libref_ufld_host.so: SHIM := $(HERE)shim_ufld
$(HERE)_ref/libref_ufld_host.so: HOSTEXTRA := -ffp-contract=off -ffunction-sections -fdata-sections -Dmain=ref_ufld_driver_main
$(HERE)_ref/libref_ufld_host.so: $(HERE)ref_wrap_ufld_host.cpp $(HERE)shim_ufld/opencv2/opencv.hpp $(HERE)shim_ufld/NvInfer.h \
                                 $(REF)/ufld/lane_det.cpp
	@mkdir -p $(HERE)_ref
	$(CXX) $(HOSTFLAGS) $(ISOLATE) -Wl,--gc-sections -I$(REF)/ufld -o $@ $<

.PHONY: ufld
