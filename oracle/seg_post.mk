# oracle/seg_post.mk -- builds (make -C oracle -f seg_post.mk; tensorrtx_b200/build.py runs it after the other oracle makefiles)
#   libseg_post_oracle.so       the CPU oracle of the YOLO segmentation post-process (seg_post_oracle.c; test infrastructure).
#                               It uses process_mask, the bilinear resize and get_rect of libtrtx_oracle.so (oracle/Makefile).
#   _ref/libref_seg_host.so     the REFERENCE's own draw_mask_bbox + scale_mask + get_rect (yolov8/src/postprocess.cpp and
#                               yolov5/src/postprocess.cpp), compiled from /root/reference where it lies, against the header
#                               shim oracle/shim_seg (a cv::Mat with storage, cv::resize = the oracle's bilinear resize,
#                               drawing calls as no-ops) by ref_wrap_seg_host.cpp.  A no-op without the reference.
CC      ?= gcc
CXX     ?= g++
REF     ?= /root/reference
HERE    := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
CFLAGS  := -O2 -fPIC -shared -ffp-contract=off -fvisibility=hidden -Wall -Wextra -std=c11 -D_GNU_SOURCE
CUDAINC := $(dir $(shell which nvcc 2>/dev/null || echo /usr/local/cuda/bin/nvcc))../include
HOSTFLAGS := -O2 -std=c++14 -fPIC -shared -w -fvisibility=hidden -ffp-contract=off -I$(HERE)shim_seg -I$(HERE)../tests/mock_trt \
             -I$(CUDAINC)

all: $(HERE)libseg_post_oracle.so ref

$(HERE)libseg_post_oracle.so: $(HERE)seg_post_oracle.c $(HERE)libtrtx_oracle.so
	$(CC) $(CFLAGS) -o $@ $< -L$(HERE) -l:libtrtx_oracle.so -Wl,-rpath,'$$ORIGIN' -lm

ifneq ($(wildcard $(REF)/yolov8/src/postprocess.cpp),)
ref: $(HERE)_ref/libref_seg_host.so
else
ref:
	@echo "reference tree not present: keeping prebuilt oracle/_ref"
endif

# the two postprocess.cpp define the same names: ref_wrap_seg_host.cpp includes each into a namespace of its own
$(HERE)_ref/seg_v8.o: $(HERE)ref_wrap_seg_host.cpp $(REF)/yolov8/src/postprocess.cpp $(HERE)shim_seg/opencv2/opencv.hpp
	@mkdir -p $(HERE)_ref
	$(CXX) $(HOSTFLAGS) -c -DREF_SEG_V8 -I$(REF)/yolov8/src -I$(REF)/yolov8/include -o $@ $<
$(HERE)_ref/seg_v5.o: $(HERE)ref_wrap_seg_host.cpp $(REF)/yolov5/src/postprocess.cpp $(HERE)shim_seg/opencv2/opencv.hpp
	@mkdir -p $(HERE)_ref
	$(CXX) $(HOSTFLAGS) -c -DREF_SEG_V5 -I$(REF)/yolov5/src -I$(REF)/yolov5/plugin -o $@ $<
# -Bsymbolic / --exclude-libs: the C++ runtime this library may carry statically must not mix with the one the Python
# process has already loaded (draw_mask_bbox's label formatting crashes otherwise)
$(HERE)_ref/libref_seg_host.so: $(HERE)_ref/seg_v8.o $(HERE)_ref/seg_v5.o $(HERE)libtrtx_oracle.so
	$(CXX) $(HOSTFLAGS) -Wl,-Bsymbolic,--exclude-libs,ALL -o $@ $(HERE)_ref/seg_v8.o $(HERE)_ref/seg_v5.o -L$(HERE) -l:libtrtx_oracle.so -Wl,-rpath,'$$ORIGIN/..'

.PHONY: all ref
