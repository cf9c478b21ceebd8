# oracle/contours.mk -- builds libcontours_oracle.so, the CPU oracle of the Mask R-CNN driver's findContours
# (contours_oracle.c; test infrastructure), with oracle/Makefile's compiler and flags.  tensorrtx_b200/build.py runs it.
include $(dir $(abspath $(lastword $(MAKEFILE_LIST))))Makefile

.DEFAULT_GOAL := contours

contours: $(HERE)libcontours_oracle.so

$(HERE)libcontours_oracle.so: $(HERE)contours_oracle.c
	$(CC) $(CFLAGS) -o $@ $<

.PHONY: contours
