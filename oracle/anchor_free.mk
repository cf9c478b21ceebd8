# oracle/anchor_free.mk -- builds, with oracle/Makefile's flags and variables (included below),
#   libanchor_free_oracle.so     the CPU oracle of yolov9's converting nms() and yolov10's get_topk (anchor_free_oracle.c), on
#                                libtrtx_oracle.so's NMS and get_rect
# and, where the reference tree is present, the REFERENCE's own code of yolov9, yolov10 and yolov13, compiled where it lies:
#   _ref/libref_af_<driver>.so       its YoloLayer plugin (plugin/yololayer.cu) with oracle/ref_wrap_anchor_free.cu;
#   _ref/libref_af_<driver>_host.so  its nms() (yolov9, yolov13) or get_topk() (yolov10) and get_rect (src/postprocess.cpp) with
#                                    oracle/ref_wrap_anchor_free_host.cpp, against oracle/shim; the drawing and mask code
#                                    nothing exported reaches is dropped (-Wl,--gc-sections).
# tensorrtx_b200.build.build_oracle() runs `make -f anchor_free.mk` after oracle/Makefile.
anchor_free:

include $(dir $(abspath $(lastword $(MAKEFILE_LIST))))Makefile

anchor_free: $(HERE)libanchor_free_oracle.so
$(HERE)libanchor_free_oracle.so: $(HERE)anchor_free_oracle.c $(HERE)libtrtx_oracle.so
	$(CC) $(CFLAGS) -o $@ $< -L$(HERE) -l:libtrtx_oracle.so -Wl,-rpath,'$$ORIGIN' -lm

AF_REF := yolov9 yolov10 yolov13
ifneq ($(wildcard $(REF)),)
anchor_free: $(foreach v,$(AF_REF),$(HERE)_ref/libref_af_$(v).so $(HERE)_ref/libref_af_$(v)_host.so)
endif
.PHONY: anchor_free

AF_BUILD = @mkdir -p $(HERE)_ref && $(NVCC) $(NVFLAGS)
$(HERE)_ref/libref_af_yolov9.so: $(HERE)ref_wrap_anchor_free.cu $(REF)/yolov9/plugin/yololayer.cu
	$(AF_BUILD) -DREF_AF_V9 -I$(REF)/yolov9/include -I$(REF)/yolov9/plugin -o $@ $^
$(HERE)_ref/libref_af_yolov10.so: $(HERE)ref_wrap_anchor_free.cu $(REF)/yolov10/plugin/yololayer.cu
	$(AF_BUILD) -I$(REF)/yolov10/include -I$(REF)/yolov10/plugin -o $@ $^
$(HERE)_ref/libref_af_yolov13.so: $(HERE)ref_wrap_anchor_free.cu $(REF)/yolov13/plugin/yololayer.cu
	$(AF_BUILD) -I$(REF)/yolov13/include -I$(REF)/yolov13/plugin -o $@ $^

$(HERE)_ref/libref_af_%_host.so: HOSTEXTRA := -ffp-contract=off -ffunction-sections -fdata-sections -DTRTX_MOCK_NO_REGISTRAR
AF_HOST = @mkdir -p $(HERE)_ref && $(CXX) $(HOSTFLAGS) $(ISOLATE) -Wl,--gc-sections
$(HERE)_ref/libref_af_yolov9_host.so: $(HERE)ref_wrap_anchor_free_host.cpp $(REF)/yolov9/src/postprocess.cpp
	$(AF_HOST) -DREF_AF_NMS -I$(REF)/yolov9/include -I$(REF)/yolov9/plugin -o $@ $^
$(HERE)_ref/libref_af_yolov10_host.so: $(HERE)ref_wrap_anchor_free_host.cpp $(REF)/yolov10/src/postprocess.cpp
	$(AF_HOST) -DREF_AF_TOPK -I$(REF)/yolov10/include -I$(REF)/yolov10/plugin -o $@ $^
$(HERE)_ref/libref_af_yolov13_host.so: $(HERE)ref_wrap_anchor_free_host.cpp $(REF)/yolov13/src/postprocess.cpp
	$(AF_HOST) -DREF_AF_NMS -I$(REF)/yolov13/include -I$(REF)/yolov13/plugin -o $@ $^
