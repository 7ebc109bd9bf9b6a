// Host-side dispatch of the fused per-(point, view) stage of the two aggregation networks: argument
// block + choice between the warpgroup kernel (view_wg.cu, the default) and the twin-warp kernel
// (view_twin.cu), which keeps an fp32 accumulator array in shared memory and is the independent
// implementation the tests compare the default against.
//
// Reference semantics: ibrnet/projection.py:103-176, ibrnet/mlp_network.py:236-284
// (dynamic) and :423-497 (static).
#include "fused_engine.cuh"
#include "geometry.cuh"
#include "nets.cuh"

namespace dyn {

// the warpgroup kernel: accumulators in registers, the fastest on an H100 (bench.py --view-kernel; DESIGN.md §3.2)
constexpr int kDefaultViewKernel = 4;

// 0 = the twin-warp kernel (view_twin.cu), 4 = the warpgroup kernel (view_wg.cu), -1 = default.
// 1 - 3 selected kernels that have been removed (the quad-schedule kernel and the sub-round pipelined
// twin kernel); launch_view_fused rejects them instead of running another kernel under their name.
static int g_view_kernel = -1;
void set_view_kernel(int which) { g_view_kernel = (which >= 0 && which <= 4) ? which : -1; }

int launch_view_fused(const dyn_net* n, ViewFusedArgs& a, int V, cudaStream_t st) {
  if (V > 16) return fail(DYN_E_INVALID, "fused per-view kernel supports V <= 16 (got %d)", V);
  a.params = n->params;
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
  switch (g_view_kernel < 0 ? kDefaultViewKernel : g_view_kernel) {
    case 0:
      if (a.tgt_idx != nullptr || a.pooled)
        return fail(DYN_E_INVALID, "the twin-warp per-view kernel (view_twin.cu) has no multi-camera form: "
                                   "select the warpgroup kernel (dyn_debug_set_view_kernel(-1))");
      return launch_view_twin(n, a, V, st);
    case 1: return fail(DYN_E_INVALID, "per-view kernel 1 (the quad-schedule kernel) has been removed");
    case 2:
    case 3:
      return fail(DYN_E_INVALID, "per-view kernel %d (the sub-round pipelined twin kernel) has been removed", g_view_kernel);
    default: return launch_view_wg(n, a, V, st);
  }
}

// host-only unit-test hooks behind dyn_debug_pack_layer / dyn_debug_tile_image_off
int debug_pack_layer(const float* W, const float* bias, int N, int Kw, int Npad, int Kpad, const int* colmap,
                     float scale, int stage_bytes, void* out_img, size_t out_bytes, size_t* img_bytes,
                     int* nchunks) {
  using namespace fe;
  if (N < 1 || Npad < N || (Npad % 16) != 0 || Npad > 256 || (Kpad % 16) != 0 || Kpad < 16 || Kw < 1 ||
      stage_bytes < Npad * 32)
    return fail(DYN_E_INVALID, "dyn_debug_pack_layer: bad shape N=%d Npad=%d Kpad=%d stage=%d", N, Npad, Kpad,
                stage_bytes);
  HostLayer L;
  L.W = W; L.N = N; L.Kw = Kw; L.Npad = Npad; L.Kpad = Kpad;
  L.colmap.assign(colmap, colmap + Kpad);
  for (int c : L.colmap)
    if (c >= Kw || c < kBiasLo) return fail(DYN_E_INVALID, "dyn_debug_pack_layer: colmap entry %d out of range", c);
  L.bias = bias; L.scale = scale;
  std::vector<uint8_t> img;
  std::vector<FusedChunk> tab;
  append_layer(L, img, tab, 0, 0, 9, true, stage_bytes);
  *img_bytes = img.size();
  *nchunks = (int)tab.size();
  if (img.size() > out_bytes) return fail(DYN_E_INVALID, "dyn_debug_pack_layer: image needs %zu bytes", img.size());
  memcpy(out_img, img.data(), img.size());
  return DYN_OK;
}
size_t debug_tile_image_off(long long row, int kgroup, int kgroups) { return fe::tile_image_off(row, kgroup, kgroups); }

}  // namespace dyn
