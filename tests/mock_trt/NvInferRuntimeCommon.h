// TEST INFRASTRUCTURE.  Forwards to the mock NvInfer.h: some reference headers (rcnn/logging.h) include the runtime header
// by its own name.
#pragma once
#include "NvInfer.h"
