# oracle/face_obb26.mk -- the reference builds of the RetinaFace / yolo26-obb post-process tests, with oracle/Makefile's
# compilers, flags and header shims (test infrastructure; tensorrtx_b200/build.py runs both):
#   _ref/libref_obb26_host.so        yolo26's own draw_bbox_obb (yolo26/src/postprocess.cpp) against shim_pose_obb
#   _ref/libref_retina_rows_host.so  retina_r50.cpp:373-388's loop on retinaface/common.hpp's get_rect_adapt_landmark
# The reference sources are compiled WHERE THEY LIE (never copied); a no-op when the reference tree is absent.
include $(dir $(abspath $(lastword $(MAKEFILE_LIST))))Makefile

FACE_OBB26 := $(HERE)_ref/libref_obb26_host.so $(HERE)_ref/libref_retina_rows_host.so
.DEFAULT_GOAL := face_obb26

ifneq ($(wildcard $(REF)),)
face_obb26: $(FACE_OBB26)
else
face_obb26:
	@echo "reference tree not present: keeping prebuilt oracle/_ref"
endif

$(HERE)_ref/libref_obb26_host.so: SHIM := $(HERE)shim_pose_obb
$(HERE)_ref/libref_obb26_host.so: HOSTEXTRA := -ffp-contract=off
$(HERE)_ref/libref_obb26_host.so: $(HERE)ref_wrap_obb26_host.cpp $(REF)/yolo26/src/postprocess.cpp \
                                  $(HERE)shim_pose_obb/opencv2/opencv.hpp
	@mkdir -p $(HERE)_ref
	$(CXX) $(HOSTFLAGS) $(ISOLATE) -I$(REF)/yolo26/src -I$(REF)/yolo26/include -o $@ $<
$(HERE)_ref/libref_retina_rows_host.so: $(HERE)ref_wrap_retina_rows_host.cpp
	@mkdir -p $(HERE)_ref
	$(CXX) $(HOSTFLAGS) -DTRTX_MOCK_NO_REGISTRAR -I$(REF)/retinaface -o $@ $<

.PHONY: face_obb26
