// SHIM -- TEST INFRASTRUCTURE.  yolov3/utils.h includes cuDNN's header and uses nothing from it.
#pragma once
