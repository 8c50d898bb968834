// device_caps.h -- properties of the target GPU that launch sizing depends on.  Plain C++ without CUDA headers, so that the
// host emulation of the element-wise kernels (tests/host_emu) compiles the same value.
#pragma once

namespace mfn {
constexpr int kNumSMs = 132;  // H100 SXM: persistent grids and grid caps are sized to one wave of CTAs on these SMs
}  // namespace mfn
