# oracle/centernet.mk -- builds, with oracle/Makefile's flags and variables (included below),
#   libcenternet_oracle.so        the CPU oracle of the CenterNet pre-process and decode (centernet_oracle.c)
#   _ref/ref_centernet.pyc        the sample's own pre_process and ctdet_decode (centernet/sample/test.py), byte-compiled
#                                 where it lies with $(PYTHON)'s py_compile, only where the reference tree is present
# tensorrtx_b200.build.build_oracle() runs `make -f centernet.mk` after oracle/Makefile, yolop.mk and detr.mk.
centernet:

include $(dir $(abspath $(lastword $(MAKEFILE_LIST))))Makefile

PYTHON ?= python3

ifneq ($(wildcard $(REF)),)
centernet: $(HERE)libcenternet_oracle.so $(HERE)_ref/ref_centernet.pyc
else
centernet: $(HERE)libcenternet_oracle.so
endif

$(HERE)libcenternet_oracle.so: $(HERE)centernet_oracle.c
	$(CC) $(CFLAGS) -o $@ $< -lm

$(HERE)_ref/ref_centernet.pyc: $(REF)/centernet/sample/test.py
	@mkdir -p $(HERE)_ref
	$(PYTHON) -c "import py_compile, sys; py_compile.compile(sys.argv[1], cfile=sys.argv[2], doraise=True)" $< $@

.PHONY: centernet
