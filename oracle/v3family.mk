# oracle/v3family.mk -- builds, with oracle/Makefile's flags and variables (included below),
#   libv3family_oracle.so          the CPU oracle of the yolov3 family's decode, each driver's box and sigmoid
#                                  (v3family_oracle.c)
# and the REFERENCE's own YoloLayer plugin of each yolov3-family driver, compiled where it lies, each with
# oracle/ref_wrap_v3_family.cu:
#   _ref/libref_v3f_yolov3.so  _ref/libref_v3f_yolov4.so  _ref/libref_v3f_csp.so  _ref/libref_v3f_tiny.so
# and the same with oracle/ref_wrap_v3_family_blob.cu too (the plugin built from a blob, on any grids and class count), in
# libraries of their own so that a test never meets a build of the first set that predates the blob entry:
#   _ref/libref_v3f_blob_<driver>.so
# and, on the host with oracle/ref_wrap_v3_family_host.cpp, the blob each one's yololayer.h constants make:
#   _ref/libref_v3f_<driver>_host.so
# and each driver's own nms() (its .cpp compiled where it lies with its main renamed, oracle/ref_wrap_v3_nms_host.cpp; the
# engine code is dropped with the sections nothing exported reaches, -Wl,--gc-sections):
#   _ref/libref_v3f_nms_<driver>.so
# (only where the reference tree is present).  Their utils.h pulls in OpenCV and dirent.h: they compile against oracle/shim_v3.
# tensorrtx_b200.build.build_oracle() runs `make -f v3family.mk` after oracle/Makefile.
v3family:

include $(dir $(abspath $(lastword $(MAKEFILE_LIST))))Makefile

v3family: $(HERE)libv3family_oracle.so
$(HERE)libv3family_oracle.so: $(HERE)v3family_oracle.c
	$(CC) $(CFLAGS) -o $@ $< -lm

V3F_REF := yolov3 yolov4 csp tiny
ifneq ($(wildcard $(REF)),)
v3family: $(foreach v,$(V3F_REF),$(HERE)_ref/libref_v3f_$(v).so $(HERE)_ref/libref_v3f_$(v)_host.so \
                                 $(HERE)_ref/libref_v3f_nms_$(v).so $(HERE)_ref/libref_v3f_blob_$(v).so)
endif
.PHONY: v3family

V3F_FLAGS = $(subst -I$(SHIM),-I$(HERE)shim_v3,$(NVFLAGS)) -DTRTX_MOCK_TRT_MAJOR=7 -DTRTX_MOCK_NO_REGISTRAR
V3F_BUILD = @mkdir -p $(HERE)_ref && $(NVCC) $(V3F_FLAGS)
$(HERE)_ref/libref_v3f_yolov3.so: $(HERE)ref_wrap_v3_family.cu $(REF)/yolov3/yololayer.cu
	$(V3F_BUILD) -I$(REF)/yolov3 -o $@ $^
$(HERE)_ref/libref_v3f_yolov4.so: $(HERE)ref_wrap_v3_family.cu $(REF)/yolov4/yololayer.cu
	$(V3F_BUILD) -I$(REF)/yolov4 -o $@ $^
$(HERE)_ref/libref_v3f_csp.so: $(HERE)ref_wrap_v3_family.cu $(REF)/scaled-yolov4/yololayer.cu
	$(V3F_BUILD) -I$(REF)/scaled-yolov4 -o $@ $^
$(HERE)_ref/libref_v3f_tiny.so: $(HERE)ref_wrap_v3_family.cu $(REF)/yolov3-tiny/yololayer.cu
	$(V3F_BUILD) -I$(REF)/yolov3-tiny -o $@ $^
V3F_BLOB := $(HERE)ref_wrap_v3_family.cu $(HERE)ref_wrap_v3_family_blob.cu
$(HERE)_ref/libref_v3f_blob_yolov3.so: $(V3F_BLOB) $(REF)/yolov3/yololayer.cu
	$(V3F_BUILD) -I$(REF)/yolov3 -o $@ $^
$(HERE)_ref/libref_v3f_blob_yolov4.so: $(V3F_BLOB) $(REF)/yolov4/yololayer.cu
	$(V3F_BUILD) -I$(REF)/yolov4 -o $@ $^
$(HERE)_ref/libref_v3f_blob_csp.so: $(V3F_BLOB) $(REF)/scaled-yolov4/yololayer.cu
	$(V3F_BUILD) -I$(REF)/scaled-yolov4 -o $@ $^
$(HERE)_ref/libref_v3f_blob_tiny.so: $(V3F_BLOB) $(REF)/yolov3-tiny/yololayer.cu
	$(V3F_BUILD) -I$(REF)/yolov3-tiny -o $@ $^

$(HERE)_ref/libref_v3f_%_host.so: SHIM := $(HERE)shim_v3
$(HERE)_ref/libref_v3f_%_host.so: HOSTEXTRA := -DTRTX_MOCK_NO_REGISTRAR -DTRTX_MOCK_TRT_MAJOR=7
V3F_HOST = @mkdir -p $(HERE)_ref && $(CXX) $(HOSTFLAGS)
$(HERE)_ref/libref_v3f_yolov3_host.so: $(HERE)ref_wrap_v3_family_host.cpp $(REF)/yolov3/yololayer.h
	$(V3F_HOST) -DREF_V3F_LEVELS=3 -I$(REF)/yolov3 -o $@ $<
$(HERE)_ref/libref_v3f_yolov4_host.so: $(HERE)ref_wrap_v3_family_host.cpp $(REF)/yolov4/yololayer.h
	$(V3F_HOST) -DREF_V3F_LEVELS=3 -I$(REF)/yolov4 -o $@ $<
$(HERE)_ref/libref_v3f_csp_host.so: $(HERE)ref_wrap_v3_family_host.cpp $(REF)/scaled-yolov4/yololayer.h
	$(V3F_HOST) -DREF_V3F_LEVELS=3 -I$(REF)/scaled-yolov4 -o $@ $<
$(HERE)_ref/libref_v3f_tiny_host.so: $(HERE)ref_wrap_v3_family_host.cpp $(REF)/yolov3-tiny/yololayer.h
	$(V3F_HOST) -DREF_V3F_LEVELS=2 -I$(REF)/yolov3-tiny -o $@ $<

V3F_NMS_DEPS := $(HERE)ref_wrap_v3_nms_host.cpp $(HERE)shim_v3/NvInfer.h $(HERE)shim_v3/cudnn.h \
                $(HERE)shim_v3/opencv2/opencv.hpp $(HERE)shim_v3/opencv2/dnn/dnn.hpp
$(HERE)_ref/libref_v3f_nms_%.so: SHIM := $(HERE)shim_v3
$(HERE)_ref/libref_v3f_nms_%.so: HOSTEXTRA := -ffp-contract=off -ffunction-sections -fdata-sections \
                                              -Dmain=ref_v3_driver_main -DTRTX_MOCK_NO_REGISTRAR -DTRTX_MOCK_TRT_MAJOR=7
V3F_NMS = @mkdir -p $(HERE)_ref && $(CXX) $(HOSTFLAGS) $(ISOLATE) -Wl,--gc-sections
$(HERE)_ref/libref_v3f_nms_yolov3.so: $(V3F_NMS_DEPS) $(REF)/yolov3/yolov3.cpp
	$(V3F_NMS) -DREF_V3_DRIVER='"yolov3.cpp"' -I$(REF)/yolov3 -o $@ $<
$(HERE)_ref/libref_v3f_nms_yolov4.so: $(V3F_NMS_DEPS) $(REF)/yolov4/yolov4.cpp
	$(V3F_NMS) -DREF_V3_DRIVER='"yolov4.cpp"' -I$(REF)/yolov4 -o $@ $<
$(HERE)_ref/libref_v3f_nms_csp.so: $(V3F_NMS_DEPS) $(REF)/scaled-yolov4/yolov4_csp.cpp $(REF)/scaled-yolov4/common.hpp
	$(V3F_NMS) -DREF_V3_CSP -DREF_V3_DRIVER='"yolov4_csp.cpp"' -I$(REF)/scaled-yolov4 -o $@ $<
$(HERE)_ref/libref_v3f_nms_tiny.so: $(V3F_NMS_DEPS) $(REF)/yolov3-tiny/yolov3-tiny.cpp
	$(V3F_NMS) -DREF_V3_DRIVER='"yolov3-tiny.cpp"' -I$(REF)/yolov3-tiny -o $@ $<
