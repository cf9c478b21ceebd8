// SHIM -- TEST INFRASTRUCTURE.  ufld/logging.h includes the runtime header; it forwards to this directory's NvInfer.h.
#pragma once
#include <NvInfer.h>
