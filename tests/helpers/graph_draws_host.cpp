// Host-side probe of the purpose-9 draws (TAG_GRAPH, graph_draw_pair in emcee_b200/csrc/philox.cuh, the header the
// kernels include), built by tests/test_graph_moves_host.py with g++ and compared with tests/graph_draws_ref.py.
#include <cmath>
#include <cstdint>
using std::cos;
using std::log;
using std::sin;
using std::sqrt;
#include "../../emcee_b200/csrc/philox.cuh"

extern "C" {
// out[r, 0 .. ndraws) for rows r < rows, as graph_move_stage_kernel fills a captured proposal's draws
void probe_graph_draws(uint64_t seed, uint64_t step, uint32_t split, int64_t rows, int normal, int64_t ndraws,
                       double* out) {
  for (int64_t i = 0; i < rows; ++i)
    for (int64_t k = 0; 2 * k < ndraws; ++k) {
      const eb::u32x4 w = eb::draw_words(seed, step, (split & 0x3Fu) | ((uint32_t)k << 6), eb::TAG_GRAPH, (uint32_t)i);
      double d0, d1;
      eb::graph_draw_pair(w, normal, d0, d1);
      out[i * ndraws + 2 * k] = d0;
      if (2 * k + 1 < ndraws) out[i * ndraws + 2 * k + 1] = d1;
    }
}
}
