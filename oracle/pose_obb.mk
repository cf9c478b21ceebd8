# oracle/pose_obb.mk -- builds (make -C oracle -f pose_obb.mk; tensorrtx_b200/build.py runs it after the other oracle makefiles)
#   _ref/libref_pose_obb_host.so  the REFERENCE's own draw_bbox_obb (get_corner) and draw_bbox_keypoints_line
#                                 (get_rect_adapt_landmark) of yolov8/src/postprocess.cpp (net 640) and
#                                 yolo11/src/postprocess.cpp (get_rect_obb, net 1024), compiled from /root/reference where
#                                 it lies, against the header shim oracle/shim_pose_obb (the drawing calls record their
#                                 points), by ref_wrap_pose_obb_host.cpp.  A no-op without the reference.
CXX     ?= g++
REF     ?= /root/reference
HERE    := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
CUDAINC := $(dir $(shell which nvcc 2>/dev/null || echo /usr/local/cuda/bin/nvcc))../include
HOSTFLAGS := -O2 -std=c++14 -fPIC -shared -w -fvisibility=hidden -ffp-contract=off -I$(HERE)shim_pose_obb \
             -I$(HERE)../tests/mock_trt -I$(CUDAINC)

all: ref

ifneq ($(wildcard $(REF)/yolov8/src/postprocess.cpp $(REF)/yolo11/src/postprocess.cpp),)
ref: $(HERE)_ref/libref_pose_obb_host.so
else
ref:
	@echo "reference tree not present: keeping prebuilt oracle/_ref"
endif

# the two postprocess.cpp define the same names: ref_wrap_pose_obb_host.cpp includes each into a namespace of its own
$(HERE)_ref/pose_obb_v8.o: $(HERE)ref_wrap_pose_obb_host.cpp $(REF)/yolov8/src/postprocess.cpp $(HERE)shim_pose_obb/opencv2/opencv.hpp
	@mkdir -p $(HERE)_ref
	$(CXX) $(HOSTFLAGS) -c -DREF_POSE_OBB_V8 -I$(REF)/yolov8/src -I$(REF)/yolov8/include -o $@ $<
$(HERE)_ref/pose_obb_v11.o: $(HERE)ref_wrap_pose_obb_host.cpp $(REF)/yolo11/src/postprocess.cpp $(HERE)shim_pose_obb/opencv2/opencv.hpp
	@mkdir -p $(HERE)_ref
	$(CXX) $(HOSTFLAGS) -c -DREF_POSE_OBB_V11 -I$(REF)/yolo11/src -I$(REF)/yolo11/include -o $@ $<
# -Bsymbolic / --exclude-libs: keep this library's C++ runtime symbols apart from the Python process's (as seg_post.mk)
$(HERE)_ref/libref_pose_obb_host.so: $(HERE)_ref/pose_obb_v8.o $(HERE)_ref/pose_obb_v11.o
	$(CXX) $(HOSTFLAGS) -Wl,-Bsymbolic,--exclude-libs,ALL -o $@ $(HERE)_ref/pose_obb_v8.o $(HERE)_ref/pose_obb_v11.o

.PHONY: all ref
