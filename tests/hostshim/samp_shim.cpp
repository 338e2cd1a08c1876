// samp_shim.cpp — test shim: the library's per-task NodesFitErrors kind (vch::fit_error_node_kinds in vc_evict.hpp, which
// ensure_evict_session derives from allocate's fit-error list) compiled by g++ for tests/test_samp_evict_cpu.py.
#include "../../volcano_b200/csrc/vc_evict.hpp"

extern "C" void vss_fit_error_node_kinds(const int32_t *fit, size_t n_fit, const int32_t *t_role, const uint32_t *r_flags,
                                         size_t T, uint8_t *out) {
  const std::vector<uint8_t> k = vch::fit_error_node_kinds(fit, n_fit, t_role, r_flags, T);
  std::copy(k.begin(), k.end(), out);
}
