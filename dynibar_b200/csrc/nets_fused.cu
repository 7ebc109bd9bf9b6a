// Host-side dispatch of the fused per-(point, view) stage of the two aggregation networks: argument
// block + choice between the warpgroup kernel (view_wg.cu, default) and the older schedules of the same work
// that keep an fp32 accumulator array in memory: the twin-warp kernel (view_twin.cu), the quad-schedule
// kernel (view_quad.cu) and the sub-round pipelined twin kernel (view_twin3.cu), kept for comparison.
//
// Reference semantics: ibrnet/projection.py:103-176, ibrnet/mlp_network.py:236-284
// (dynamic) and :423-497 (static).
#include <stdlib.h>

#include "fused_engine.cuh"
#include "geometry.cuh"
#include "nets.cuh"

namespace dyn {

// the warpgroup kernel: accumulators in registers, the fastest on an H100 (bench.py --view-kernel; DESIGN.md §3.2)
constexpr int kDefaultViewKernel = 4;

// Schedules of the same per-tile work: 0 = the twin-warp kernel (view_twin.cu: one CTA per SM, one tile),
// 1 = the quad kernel (view_quad.cu: one CTA per SM alternating between two tiles), 2 = the twin-warp kernel
// with sub-round pipelined layers (view_twin3.cu; 3 = the same with one barrier arrival per warp), 4 = the
// warpgroup kernel (view_wg.cu).  DYN_VIEW_KERNEL=twin|quad|pipe or dyn_debug_set_view_kernel(); -1 = default.
static int g_view_kernel = -1;
void set_view_kernel(int which) { g_view_kernel = (which >= 0 && which <= 4) ? which : -1; }
static int view_kernel() {
  if (g_view_kernel < 0) {
    const char* e = getenv("DYN_VIEW_KERNEL");
    const char c = e == nullptr ? 0 : e[0];
    g_view_kernel = c == 't' ? 0 : (c == 'q' ? 1 : (c == 'p' ? 2 : (c == 'e' ? 3 : kDefaultViewKernel)));
  }
  return g_view_kernel;
}

bool use_twin_chains() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("DYN_CHAINS");
    v = (e != nullptr && e[0] == 'f') ? 0 : 1;
  }
  return v == 1;
}

int producer_lanes() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("DYN_PRODUCERS");
    v = (e != nullptr && e[0] == '2') ? 2 : 1;
  }
  return v;
}

int launch_view_fused(const dyn_net* n, ViewFusedArgs& a, int V, cudaStream_t st) {
  if (V > 16) return fail(DYN_E_INVALID, "fused per-view kernel supports V <= 16 (got %d)", V);
  a.params = n->params;
  a.producers = producer_lanes();
  const bool st_net = n->kind == DYN_NET_STATIC;
  if (st_net) {
    const StaticLayout& L = n->sl;
    a.o_b1 = L.ray_dir0.b; a.o_b2 = L.ray_dir2.b; a.o_b3 = L.base0.b; a.o_b4 = L.base2.b;
    a.o_b5 = L.vis0.b; a.o_b6 = L.vis2.b; a.o_w6 = L.vis2.w; a.o_b7 = L.vis2_0.b;
    a.o_w8 = L.vis2_2.w; a.o_b8 = L.vis2_2.b; a.o_s = L.s;
    a.anti_alias = n->anti_alias; a.mask_rgb = n->mask_rgb;
  } else {
    const DynamicLayout& L = n->dl;
    a.o_b1 = 0; a.o_b2 = 0; a.o_b3 = L.base0.b; a.o_b4 = L.base2.b;
    a.o_b5 = L.vis0.b; a.o_b6 = L.vis2.b; a.o_w6 = L.vis2.w; a.o_b7 = L.vis2_0.b;
    a.o_w8 = L.vis2_2.w; a.o_b8 = L.vis2_2.b; a.o_s = -1;
    a.anti_alias = 0; a.mask_rgb = 0;
  }
  switch (view_kernel()) {
    case 1: return launch_view_quad(n, a, V, st);
    case 2: return launch_view_twin3(n, a, V, st, false);
    case 3: return launch_view_twin3(n, a, V, st, true);  // + one barrier arrival per warp ("elected")
    case 4: return launch_view_wg(n, a, V, st);
    default: return launch_view_twin(n, a, V, st);
  }
}

}  // namespace dyn
