// NVTX ranges for timelines (nsys / ncu range filtering).  Header-only NVTX v3: no library to link;
// when no tool is attached the calls are no-ops.  The reference has no tracing beyond
// `set -o xtrace` in its sweep scripts.
#pragma once

#include <nvtx3/nvToolsExt.h>

#include <string>

namespace hpcp {

struct NvtxRange {
  explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
  explicit NvtxRange(const std::string& name) { nvtxRangePushA(name.c_str()); }
  ~NvtxRange() { nvtxRangePop(); }
  NvtxRange(const NvtxRange&) = delete;
  NvtxRange& operator=(const NvtxRange&) = delete;
};

}  // namespace hpcp
