# oracle/rcnn_pre.mk -- builds (make -C oracle -f rcnn_pre.mk; tensorrtx_b200/build.py runs it after oracle/Makefile)
#   librcnn_pre_oracle.so        the CPU oracle of the Mask R-CNN pre-process (rcnn_pre_oracle.c; test infrastructure).
#   _ref/libref_rcnn_pre_host.so the REFERENCE's preprocessImg (rcnn/common.hpp:79-110), compiled from /root/reference where it
#                                lies, against tests/mock_trt and the recording header shim oracle/shim_rcnn_pre.  A no-op
#                                without the reference.
CC      ?= gcc
CXX     ?= g++
REF     ?= /root/reference
HERE    := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
CFLAGS  := -O2 -fPIC -shared -ffp-contract=off -fvisibility=hidden -Wall -Wextra -std=c11 -D_GNU_SOURCE
CUDAINC := $(dir $(shell which nvcc 2>/dev/null || echo /usr/local/cuda/bin/nvcc))../include
HOSTFLAGS := -O2 -std=c++14 -fPIC -shared -w -fvisibility=hidden -I$(HERE)shim_rcnn_pre -I$(HERE)../tests/mock_trt -I$(CUDAINC)

all: $(HERE)librcnn_pre_oracle.so ref

$(HERE)librcnn_pre_oracle.so: $(HERE)rcnn_pre_oracle.c
	$(CC) $(CFLAGS) -o $@ $< -lm

ifneq ($(wildcard $(REF)/rcnn/common.hpp),)
ref: $(HERE)_ref/libref_rcnn_pre_host.so
else
ref:
	@echo "reference tree not present: keeping prebuilt oracle/_ref"
endif

$(HERE)_ref/libref_rcnn_pre_host.so: $(HERE)ref_wrap_rcnn_pre_host.cpp $(HERE)shim_rcnn_pre/opencv2/opencv.hpp
	@mkdir -p $(HERE)_ref
	$(CXX) $(HOSTFLAGS) -I$(REF)/rcnn -o $@ $<

.PHONY: all ref
