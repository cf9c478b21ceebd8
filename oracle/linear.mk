# oracle/linear.mk -- builds, with oracle/Makefile's flags and variables (included below),
#   liblinear_oracle.so           the CPU oracle of the bilinear letterbox pre-process of yolov3, yolov4, scaled-yolov4,
#                                 yolov3-spp and RetinaFace, and of their get_rect (linear_oracle.c, on cls_oracle.c's resize)
#   _ref/libref_v3_<driver>.so    the get_rect of yolov3, yolov4, scaled-yolov4 (csp), yolov3-tiny and yolov3-spp, and
#                                 yolov3-spp's letterbox, compiled where they lie (only where the reference tree is present)
# tensorrtx_b200.build.build_oracle() runs `make -f linear.mk` after oracle/Makefile and the other oracle makefiles.
linear:

include $(dir $(abspath $(lastword $(MAKEFILE_LIST))))Makefile

linear: $(HERE)liblinear_oracle.so

$(HERE)liblinear_oracle.so: $(HERE)linear_oracle.c $(HERE)cls_oracle.c
	$(CC) $(CFLAGS) -o $@ $< -lm

.PHONY: linear

# Each driver's own get_rect (yolov3, yolov4, scaled-yolov4 via its common.hpp, yolov3-tiny, yolov3-spp) and yolov3-spp's own
# letterbox, compiled where they lie against shim_v3 with their main renamed; the drivers' engine code is dropped with the
# sections nothing exported reaches (-Wl,--gc-sections), and with it every reference to TensorRT and CUDA entry points.
V3_REF  := yolov3 yolov4 csp tiny spp
V3_DEPS := $(HERE)ref_wrap_v3_host.cpp $(HERE)shim_v3/NvInfer.h $(HERE)shim_v3/cudnn.h $(HERE)shim_v3/opencv2/opencv.hpp \
           $(HERE)shim_v3/opencv2/dnn/dnn.hpp
ifneq ($(wildcard $(REF)),)
linear: $(foreach v,$(V3_REF),$(HERE)_ref/libref_v3_$(v).so)
endif
$(HERE)_ref/libref_v3_%.so: SHIM := $(HERE)shim_v3
$(HERE)_ref/libref_v3_%.so: HOSTEXTRA := -ffp-contract=off -ffunction-sections -fdata-sections -Dmain=ref_v3_driver_main \
                                         -DTRTX_MOCK_NO_REGISTRAR -DTRTX_MOCK_TRT_MAJOR=7
V3_BUILD = @mkdir -p $(HERE)_ref && $(CXX) $(HOSTFLAGS) $(ISOLATE) -Wl,--gc-sections
$(HERE)_ref/libref_v3_yolov3.so: $(V3_DEPS) $(REF)/yolov3/yolov3.cpp
	$(V3_BUILD) -DREF_V3_DRIVER='"yolov3.cpp"' -I$(REF)/yolov3 -o $@ $<
$(HERE)_ref/libref_v3_yolov4.so: $(V3_DEPS) $(REF)/yolov4/yolov4.cpp
	$(V3_BUILD) -DREF_V3_DRIVER='"yolov4.cpp"' -I$(REF)/yolov4 -o $@ $<
$(HERE)_ref/libref_v3_csp.so: $(V3_DEPS) $(REF)/scaled-yolov4/yolov4_csp.cpp $(REF)/scaled-yolov4/common.hpp
	$(V3_BUILD) -DREF_V3_DRIVER='"yolov4_csp.cpp"' -I$(REF)/scaled-yolov4 -o $@ $<
$(HERE)_ref/libref_v3_tiny.so: $(V3_DEPS) $(REF)/yolov3-tiny/yolov3-tiny.cpp
	$(V3_BUILD) -DREF_V3_DRIVER='"yolov3-tiny.cpp"' -I$(REF)/yolov3-tiny -o $@ $<
$(HERE)_ref/libref_v3_spp.so: $(V3_DEPS) $(REF)/yolov3-spp/yolov3-spp.cpp
	$(V3_BUILD) -DREF_V3_SPP -DREF_V3_DRIVER='"yolov3-spp.cpp"' -I$(REF)/yolov3-spp -o $@ $<
