# oracle/refinedet.mk -- builds, with oracle/Makefile's flags and variables (included below),
#   librefinedet_oracle.so        the CPU oracle of the RefineDet pre- and post-process (refinedet_oracle.c, on cls_oracle.c's
#                                 resize)
# The reference's post-process is libtorch code, and its driver loop sits inside main(), so no reference library is built.
# tensorrtx_b200.build.build_oracle() runs `make -f refinedet.mk` after the other oracle makefiles.
refinedet:

include $(dir $(abspath $(lastword $(MAKEFILE_LIST))))Makefile

refinedet: $(HERE)librefinedet_oracle.so

$(HERE)librefinedet_oracle.so: $(HERE)refinedet_oracle.c $(HERE)cls_oracle.c
	$(CC) $(CFLAGS) -o $@ $< -lm

.PHONY: refinedet
