# oracle/cubic.mk -- builds, with oracle/Makefile's flags and variables (included below),
#   libcubic_oracle.so            the CPU oracle of the bicubic letterbox pre-process of yolov3-tiny and retinafaceAntiCov
#                                 (cubic_oracle.c)
# Both drivers' preprocess_img and plane loops sit next to their engine calls, so no reference library is built for them.
# tensorrtx_b200.build.build_oracle() runs `make -f cubic.mk` after oracle/Makefile and the other oracle makefiles.
cubic:

include $(dir $(abspath $(lastword $(MAKEFILE_LIST))))Makefile

cubic: $(HERE)libcubic_oracle.so

$(HERE)libcubic_oracle.so: $(HERE)cubic_oracle.c
	$(CC) $(CFLAGS) -o $@ $< -lm

.PHONY: cubic
