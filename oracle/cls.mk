# oracle/cls.mk -- the YOLO classification pre- and post-process tests' builds, with oracle/Makefile's compilers, flags and
# header shims (test infrastructure; tensorrtx_b200/build.py runs it):
#   libcls_oracle.so               the CPU oracle (cls_oracle.c)
#   _ref/libref_cls_<driver>.so    each cls driver's own batch_preprocess, softmax and topk (yolov8_cls.cpp, yolo11_cls.cpp,
#                                  yolov5_cls.cpp, yolo26_cls.cpp), compiled where it lies against shim_cls, its main renamed
# A no-op for _ref when the reference tree is absent.
include $(dir $(abspath $(lastword $(MAKEFILE_LIST))))Makefile

CLS_REF := $(HERE)_ref/libref_cls_yolov8.so $(HERE)_ref/libref_cls_yolo11.so $(HERE)_ref/libref_cls_yolov5.so \
           $(HERE)_ref/libref_cls_yolo26.so
.DEFAULT_GOAL := cls

ifneq ($(wildcard $(REF)),)
cls: $(HERE)libcls_oracle.so $(CLS_REF)
else
cls: $(HERE)libcls_oracle.so
	@echo "reference tree not present: keeping prebuilt oracle/_ref"
endif

$(HERE)libcls_oracle.so: $(HERE)cls_oracle.c
	$(CC) $(CFLAGS) -o $@ $< -lm

# the drivers' unused engine code is dropped with the sections nothing exported reaches (-Wl,--gc-sections), and with it
# every reference to TensorRT and CUDA entry points this image has no library for
$(CLS_REF): SHIM := $(HERE)shim_cls
$(CLS_REF): HOSTEXTRA := -ffp-contract=off -ffunction-sections -fdata-sections -Dmain=ref_cls_driver_main
CLS_DEPS := $(HERE)ref_wrap_cls_host.cpp $(HERE)shim_cls/opencv2/opencv.hpp $(HERE)shim_cls/NvInfer.h
$(HERE)_ref/libref_cls_yolov8.so: $(CLS_DEPS) $(REF)/yolov8/yolov8_cls.cpp
	@mkdir -p $(HERE)_ref
	$(CXX) $(HOSTFLAGS) $(ISOLATE) -Wl,--gc-sections -DREF_CLS_SOFTMAX -DREF_CLS_DRIVER='"yolov8_cls.cpp"' -I$(REF)/yolov8 \
	    -I$(REF)/yolov8/include -o $@ $<
$(HERE)_ref/libref_cls_yolo11.so: $(CLS_DEPS) $(REF)/yolo11/yolo11_cls.cpp
	@mkdir -p $(HERE)_ref
	$(CXX) $(HOSTFLAGS) $(ISOLATE) -Wl,--gc-sections -DREF_CLS_SOFTMAX -DREF_CLS_DRIVER='"yolo11_cls.cpp"' -I$(REF)/yolo11 \
	    -I$(REF)/yolo11/include -o $@ $<
$(HERE)_ref/libref_cls_yolov5.so: $(CLS_DEPS) $(REF)/yolov5/yolov5_cls.cpp
	@mkdir -p $(HERE)_ref
	$(CXX) $(HOSTFLAGS) $(ISOLATE) -Wl,--gc-sections -DREF_CLS_SOFTMAX -DREF_CLS_V5 -DREF_CLS_DRIVER='"yolov5_cls.cpp"' \
	    -I$(REF)/yolov5 -I$(REF)/yolov5/src -o $@ $<
$(HERE)_ref/libref_cls_yolo26.so: $(CLS_DEPS) $(REF)/yolo26/yolo26_cls.cpp
	@mkdir -p $(HERE)_ref
	$(CXX) $(HOSTFLAGS) $(ISOLATE) -Wl,--gc-sections -DTRTX_MOCK_NO_REGISTRAR -DREF_CLS_DRIVER='"yolo26_cls.cpp"' -I$(REF)/yolo26 \
	    -I$(REF)/yolo26/include -I$(REF)/yolo26/plugin -o $@ $<

.PHONY: cls
