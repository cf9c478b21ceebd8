# oracle/detr.mk -- builds, with oracle/Makefile's flags and variables (included below),
#   libdetr_oracle.so             the CPU oracle of the DETR pre- and post-process (detr_oracle.c, on cls_oracle.c's resize)
# DETR's post loop sits inside its driver's main(), so no reference library is built for it.
# tensorrtx_b200.build.build_oracle() runs `make -f detr.mk` after oracle/Makefile and yolop.mk.
detr:

include $(dir $(abspath $(lastword $(MAKEFILE_LIST))))Makefile

detr: $(HERE)libdetr_oracle.so

$(HERE)libdetr_oracle.so: $(HERE)detr_oracle.c $(HERE)cls_oracle.c
	$(CC) $(CFLAGS) -o $@ $< -lm

.PHONY: detr
