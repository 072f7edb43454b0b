// b2r_torch.cpp -- compiled torch binding of the eager drop-in path.
//
// `GaussianRasterizer.forward` (exavatar_release_b200/rasterizer.py; reference call site avatar/common/nets/module.py:632-640)
// spent ~0.2 ms of Python per render around ~0.1 ms of kernel launches: building ctypes structs, a dozen torch.empty calls,
// the autograd.Function trampolines in both directions (tools/eager_profile.py).  This file is the same
// host logic -- argument normalisation, the duplicate-capacity policy with its pinned-host status mirror, workspace
// allocation, the saved context, the backward call -- as a C++ torch::autograd::Function over the SAME C ABI
// (include/b200raster.h, libb200raster.so).  No kernels here and no second implementation of anything on the device.
//
// Scope: the plain (un-skinned) rasteriser call with adaptive capacity.  rasterizer.py keeps the Python route for
// debug=True (snapshot dump on failure), fixed-capacity / CUDA-graph capture, statistics requests and fused skinning.
#include <torch/extension.h>

#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>
#include <cuda_runtime.h>

#include <chrono>
#include <map>
#include <memory>
#include <mutex>
#include <tuple>

#include "b200raster.h"

namespace {

using torch::autograd::AutogradContext;
using torch::autograd::variable_list;

struct DeviceState {
  std::mutex mu;
  volatile uint64_t* mirror = nullptr;  // 2 x uint64 pinned host memory: {num_dups, token}
  uint64_t token = 0;
  std::map<std::tuple<int64_t, int64_t, int64_t>, uint64_t> predicted;  // (P, W, H) -> last duplicate count
};

DeviceState& state_of(int device) {
  static std::mutex mu;
  static std::map<int, std::unique_ptr<DeviceState>> states;
  std::lock_guard<std::mutex> g(mu);
  auto& s = states[device];
  if (!s) {
    s = std::make_unique<DeviceState>();
    void* p = nullptr;
    TORCH_CHECK(cudaHostAlloc(&p, 2 * sizeof(uint64_t), cudaHostAllocPortable) == cudaSuccess,
                "b200raster: cannot allocate the pinned status mirror");
    s->mirror = static_cast<volatile uint64_t*>(p);
    s->mirror[0] = 0;
    s->mirror[1] = 0;
  }
  return *s;
}

void check(int rc, const char* what) {
  TORCH_CHECK(rc == B2R_OK, "b200raster: ", what, " failed: ", b2r_strerror(rc), " (cuda error ", b2r_last_cuda_error(), ")");
}

// spin until the scan kernel has published {num_dups, token}
uint64_t wait_mirror(DeviceState& st, uint64_t token, cudaStream_t stream) {
  const auto t0 = std::chrono::steady_clock::now();
  uint64_t spins = 0;
  while (st.mirror[1] != token) {
    if ((++spins & 0xfffff) == 0 && std::chrono::steady_clock::now() - t0 > std::chrono::seconds(20)) {
      cudaStreamSynchronize(stream);  // surfaces a sticky CUDA error if the kernels died
      TORCH_CHECK(st.mirror[1] == token, "b200raster: projection phase never published its duplicate count");
    }
  }
  return st.mirror[0];
}

at::Tensor f32c(const at::Tensor& t, const char* name) {
  TORCH_CHECK(t.is_cuda(), "b200raster: `", name, "` must be a CUDA tensor (got ", t.device(), "); there is no CPU fallback");
  return (t.scalar_type() == at::kFloat ? t : t.to(at::kFloat)).contiguous();
}
bool present(const c10::optional<at::Tensor>& t) { return t.has_value() && t->defined() && t->numel() > 0; }
const float* fptr(const at::Tensor& t) { return t.defined() && t.numel() > 0 ? t.data_ptr<float>() : nullptr; }

B2RScene make_scene(int64_t P, int64_t H, int64_t W, int64_t sh_degree, uint32_t flags, double scale_modifier, double tanfovx,
                    double tanfovy, const at::Tensor& bg, const at::Tensor& view, const at::Tensor& proj,
                    const at::Tensor& campos, const at::Tensor& means3D, const at::Tensor& shs, const at::Tensor& colors,
                    const at::Tensor& opac, const at::Tensor& scales, const at::Tensor& rots, const at::Tensor& cov) {
  B2RScene sc{};
  sc.P = (int32_t)P;
  sc.width = (int32_t)W;
  sc.height = (int32_t)H;
  sc.sh_degree = (int32_t)sh_degree;
  sc.sh_coeffs = shs.defined() && shs.numel() > 0 ? (int32_t)shs.size(1) : 0;
  sc.flags = flags;
  sc.scale_modifier = (float)scale_modifier;
  sc.tanfovx = (float)tanfovx;
  sc.tanfovy = (float)tanfovy;
  sc.bg = fptr(bg);
  sc.viewmatrix = fptr(view);
  sc.projmatrix = fptr(proj);
  sc.campos = fptr(campos);
  sc.means3D = fptr(means3D);
  sc.shs = fptr(shs);
  sc.colors_precomp = fptr(colors);
  sc.opacities = fptr(opac);
  sc.scales = fptr(scales);
  sc.rotations = fptr(rots);
  sc.cov3D_precomp = fptr(cov);
  return sc;
}

struct RasterizeFn : public torch::autograd::Function<RasterizeFn> {
  // tensor inputs first (their gradients are returned in this order), then the settings
  static variable_list forward(AutogradContext* ctx, const at::Tensor& means3D_in, const at::Tensor& means2D,
                               const c10::optional<at::Tensor>& sh_in, const c10::optional<at::Tensor>& colors_in,
                               const at::Tensor& opac_in, const c10::optional<at::Tensor>& scales_in,
                               const c10::optional<at::Tensor>& rots_in, const c10::optional<at::Tensor>& cov_in, int64_t H,
                               int64_t W, double tanfovx, double tanfovy, const at::Tensor& bg_in, double scale_modifier,
                               const at::Tensor& view_in, const at::Tensor& proj_in, int64_t sh_degree,
                               const at::Tensor& campos_in, bool tile_cull, bool speculative, double headroom,
                               bool segmented) {
    const bool need_grad = means3D_in.requires_grad() || means2D.requires_grad() || (present(sh_in) && sh_in->requires_grad()) ||
                           (present(colors_in) && colors_in->requires_grad()) || opac_in.requires_grad() ||
                           (present(scales_in) && scales_in->requires_grad()) ||
                           (present(rots_in) && rots_in->requires_grad()) || (present(cov_in) && cov_in->requires_grad());
    const at::Tensor means3D = f32c(means3D_in, "means3D");
    const at::Tensor shs = present(sh_in) ? f32c(*sh_in, "shs") : at::Tensor();
    const at::Tensor colors = present(colors_in) ? f32c(*colors_in, "colors_precomp") : at::Tensor();
    const at::Tensor opac = f32c(opac_in, "opacities");
    const at::Tensor scales = present(scales_in) ? f32c(*scales_in, "scales") : at::Tensor();
    const at::Tensor rots = present(rots_in) ? f32c(*rots_in, "rotations") : at::Tensor();
    const at::Tensor cov = present(cov_in) ? f32c(*cov_in, "cov3D_precomp") : at::Tensor();
    const auto dev = means3D.device();
    c10::cuda::CUDAGuard guard(dev);
    const cudaStream_t stream = c10::cuda::getCurrentCUDAStream(dev.index()).stream();
    const int64_t P = means3D.size(0);
    const auto f32 = means3D.options().dtype(at::kFloat);
    const auto u8 = means3D.options().dtype(at::kByte);
    const auto i32 = means3D.options().dtype(at::kInt);
    at::Tensor color = at::empty({3, H, W}, f32), depth = at::empty({1, H, W}, f32), alpha = at::empty({1, H, W}, f32);
    at::Tensor radii = at::empty({P}, i32);
    ctx->set_materialize_grads(false);  // unused outputs (depth, alpha) arrive as undefined, not as zero images
    ctx->saved_data["P"] = P;
    ctx->saved_data["m2_shape"] = means2D.sizes().vec();
    ctx->saved_data["op_shape"] = opac_in.sizes().vec();
    ctx->saved_data["m3_shape"] = means3D_in.sizes().vec();
    if (P == 0) {  // upstream returns a zero image without launching anything
      color.zero_(); depth.zero_(); alpha.zero_();
      ctx->mark_non_differentiable({radii});
      return {color, radii, depth, alpha};
    }
    const at::Tensor bg = f32c(bg_in.to(dev), "bg"), view = f32c(view_in.to(dev), "viewmatrix");
    const at::Tensor proj = f32c(proj_in.to(dev), "projmatrix"), campos = f32c(campos_in.to(dev), "campos");
    const uint32_t flags = tile_cull ? 0u : B2R_FLAG_NO_TILE_CULL;
    const B2RScene sc = make_scene(P, H, W, sh_degree, flags, scale_modifier, tanfovx, tanfovy, bg, view, proj, campos,
                                   means3D, shs, colors, opac, scales, rots, cov);
    const size_t ctx_bytes = b2r_ctx_bytes((int32_t)P, (int32_t)W, (int32_t)H);
    at::Tensor ctx_buf = at::empty({(int64_t)ctx_bytes}, u8);
    B2RForwardOutputs out{color.data_ptr<float>(), depth.data_ptr<float>(), alpha.data_ptr<float>(), radii.data_ptr<int32_t>()};

    DeviceState& st = state_of(dev.index());
    at::Tensor ids, ck;
    uint64_t cap = 0, num = 0;
    auto workspace = [&](uint64_t capacity, uint64_t token) {
      cap = capacity;
      ids = at::empty({(int64_t)std::max<uint64_t>(cap, 1)}, i32);
      const size_t sbytes = b2r_scratch_bytes((int32_t)P, (int32_t)W, (int32_t)H, cap);
      at::Tensor scratch = at::empty({(int64_t)sbytes}, u8);  // recycled by the caching allocator in stream order
      size_t ckb = 0;
      ck = at::Tensor();
      if (need_grad && segmented) {
        ckb = b2r_checkpoint_bytes((int32_t)W, (int32_t)H, cap);
        ck = at::empty({(int64_t)ckb}, u8);
      }
      B2RWorkspace ws{ctx_buf.data_ptr(), ctx_bytes, (uint32_t*)ids.data_ptr<int32_t>(), cap, scratch.data_ptr(), sbytes,
                      const_cast<uint64_t*>(st.mirror), token, ck.defined() ? ck.data_ptr() : nullptr, ckb};
      return ws;
    };
    {
      std::lock_guard<std::mutex> g(st.mu);
      const auto key = std::make_tuple(P, W, H);
      const auto it = st.predicted.find(key);
      if (speculative && it != st.predicted.end()) {
        uint64_t token = ++st.token;
        B2RWorkspace ws = workspace((uint64_t)((double)it->second * headroom) + 4096, token);
        check(b2r_forward(&sc, &ws, &out, stream), "b2r_forward");
        num = wait_mirror(st, token, stream);
        if (num > cap) {  // misprediction: the whole forward again with the exact size
          token = ++st.token;
          ws = workspace(num, token);
          check(b2r_forward(&sc, &ws, &out, stream), "b2r_forward");
          num = wait_mirror(st, token, stream);
        }
      } else {
        const uint64_t token = ++st.token;
        B2RWorkspace ws0{ctx_buf.data_ptr(), ctx_bytes, nullptr, 0, nullptr, 0, const_cast<uint64_t*>(st.mirror), token,
                         nullptr, 0};
        check(b2r_forward_project(&sc, &ws0, radii.data_ptr<int32_t>(), stream), "b2r_forward_project");
        num = wait_mirror(st, token, stream);
        B2RWorkspace ws = workspace(num, token);
        check(b2r_forward_render(&sc, &ws, &out, stream), "b2r_forward_render");
      }
      st.predicted[key] = num;
    }
    // what must survive until backward (SURVEY.md section 8b "Ownership"); undefined tensors are saved as such
    ctx->save_for_backward({means3D, shs, colors, opac, scales, rots, cov, bg, view, proj, campos, ctx_buf, ids, ck});
    ctx->saved_data["H"] = H;
    ctx->saved_data["W"] = W;
    ctx->saved_data["tanfovx"] = tanfovx;
    ctx->saved_data["tanfovy"] = tanfovy;
    ctx->saved_data["scale_modifier"] = scale_modifier;
    ctx->saved_data["sh_degree"] = sh_degree;
    ctx->saved_data["flags"] = (int64_t)flags;
    ctx->saved_data["cap"] = (int64_t)cap;
    ctx->mark_non_differentiable({radii});
    return {color, radii, depth, alpha};
  }

  static variable_list backward(AutogradContext* ctx, variable_list grads) {
    // one entry per forward argument: 8 tensors, then 14 settings
    variable_list out(22);
    at::Tensor g_color = grads[0], g_depth = grads[2], g_alpha = grads[3];
    if (!g_color.defined() && !g_depth.defined() && !g_alpha.defined()) return out;
    const int64_t P = ctx->saved_data["P"].toInt();
    const auto m2_shape = ctx->saved_data["m2_shape"].toIntVector();
    const auto op_shape = ctx->saved_data["op_shape"].toIntVector();
    const auto m3_shape = ctx->saved_data["m3_shape"].toIntVector();
    if (!g_color.defined()) {  // only depth / alpha were used downstream
      const at::Tensor& ref = g_depth.defined() ? g_depth : g_alpha;
      g_color = at::zeros({3, ref.size(-2), ref.size(-1)}, ref.options().dtype(at::kFloat));
    }
    if (P == 0) {
      const auto o = g_color.options().dtype(at::kFloat);
      out[0] = at::zeros(m3_shape, o);
      out[1] = at::zeros(m2_shape, o);
      out[4] = at::zeros(op_shape, o);
      return out;
    }
    const auto sv = ctx->get_saved_variables();
    const at::Tensor &means3D = sv[0], &shs = sv[1], &colors = sv[2], &opac = sv[3], &scales = sv[4], &rots = sv[5],
                     &cov = sv[6], &bg = sv[7], &view = sv[8], &proj = sv[9], &campos = sv[10], &ctx_buf = sv[11],
                     &ids = sv[12], &ck = sv[13];
    const int64_t H = ctx->saved_data["H"].toInt(), W = ctx->saved_data["W"].toInt();
    const auto dev = means3D.device();
    c10::cuda::CUDAGuard guard(dev);
    const cudaStream_t stream = c10::cuda::getCurrentCUDAStream(dev.index()).stream();
    const B2RScene sc = make_scene(P, H, W, ctx->saved_data["sh_degree"].toInt(), (uint32_t)ctx->saved_data["flags"].toInt(),
                                   ctx->saved_data["scale_modifier"].toDouble(), ctx->saved_data["tanfovx"].toDouble(),
                                   ctx->saved_data["tanfovy"].toDouble(), bg, view, proj, campos, means3D, shs, colors, opac,
                                   scales, rots, cov);
    const auto f32 = means3D.options().dtype(at::kFloat);
    const int64_t M = sc.sh_coeffs;
    at::Tensor d_means3D = at::empty({P, 3}, f32), d_means2D = at::empty({P, 3}, f32), d_colors = at::empty({P, 3}, f32);
    at::Tensor d_opac = at::empty({P, 1}, f32), d_scales = at::empty({P, 3}, f32), d_rots = at::empty({P, 4}, f32);
    at::Tensor d_cov = at::empty({P, 6}, f32);
    at::Tensor d_shs = M > 0 ? at::empty({P, M, 3}, f32) : at::Tensor();
    g_color = f32c(g_color, "grad_color");
    if (g_depth.defined()) g_depth = f32c(g_depth, "grad_depth");
    if (g_alpha.defined()) g_alpha = f32c(g_alpha, "grad_alpha");
    const size_t sbytes = b2r_backward_scratch_bytes((int32_t)P);
    at::Tensor scratch = at::empty({(int64_t)sbytes}, means3D.options().dtype(at::kByte));
    B2RWorkspace ws{ctx_buf.data_ptr(), (size_t)ctx_buf.numel(), (uint32_t*)ids.data_ptr<int32_t>(),
                    (uint64_t)ctx->saved_data["cap"].toInt(), nullptr, 0, nullptr, 0,
                    ck.defined() ? ck.data_ptr() : nullptr, ck.defined() ? (size_t)ck.numel() : 0};
    B2RBackwardArgs a{};
    a.dL_dcolor = fptr(g_color);
    a.dL_ddepth = fptr(g_depth);
    a.dL_dalpha = fptr(g_alpha);
    a.dL_dmeans3D = d_means3D.data_ptr<float>();
    a.dL_dmeans2D = d_means2D.data_ptr<float>();
    a.dL_dshs = d_shs.defined() ? d_shs.data_ptr<float>() : nullptr;
    a.dL_dcolors = d_colors.data_ptr<float>();
    a.dL_dopacities = d_opac.data_ptr<float>();
    a.dL_dscales = d_scales.data_ptr<float>();
    a.dL_drotations = d_rots.data_ptr<float>();
    a.dL_dcov3D = d_cov.data_ptr<float>();
    check(b2r_backward(&sc, &ws, &a, scratch.data_ptr(), sbytes, stream), "b2r_backward");
    int64_t m2_numel = 1;
    for (auto v : m2_shape) m2_numel *= v;
    out[0] = d_means3D;
    out[1] = m2_numel == P * 3 ? d_means2D.reshape(m2_shape) : d_means2D;
    if (shs.defined()) out[2] = d_shs;
    if (colors.defined()) out[3] = d_colors;
    out[4] = d_opac.reshape(op_shape);
    if (scales.defined()) out[5] = d_scales;
    if (rots.defined()) out[6] = d_rots;
    if (cov.defined()) out[7] = d_cov;
    return out;
  }
};

std::vector<at::Tensor> rasterize(const at::Tensor& means3D, const at::Tensor& means2D, const c10::optional<at::Tensor>& sh,
                                  const c10::optional<at::Tensor>& colors, const at::Tensor& opac,
                                  const c10::optional<at::Tensor>& scales, const c10::optional<at::Tensor>& rots,
                                  const c10::optional<at::Tensor>& cov, int64_t H, int64_t W, double tanfovx, double tanfovy,
                                  const at::Tensor& bg, double scale_modifier, const at::Tensor& view, const at::Tensor& proj,
                                  int64_t sh_degree, const at::Tensor& campos, bool tile_cull, bool speculative,
                                  double headroom, bool segmented) {
  return RasterizeFn::apply(means3D, means2D, sh, colors, opac, scales, rots, cov, H, W, tanfovx, tanfovy, bg, scale_modifier,
                            view, proj, sh_degree, campos, tile_cull, speculative, headroom, segmented);
}

}  // namespace

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.def("rasterize", &rasterize, "GaussianRasterizer forward with autograd (compiled host path over libb200raster.so)");
  m.def("abi_version", []() { return b2r_abi_version(); });
  m.def("get_predicted", [](int64_t device, int64_t P, int64_t W, int64_t H) -> int64_t {  // -1: shape not seen yet
    DeviceState& st = state_of((int)device);
    std::lock_guard<std::mutex> g(st.mu);
    const auto it = st.predicted.find(std::make_tuple(P, W, H));
    return it == st.predicted.end() ? -1 : (int64_t)it->second;
  });
  // tests: plant a capacity prediction (a wrong one must be repaired transparently by the forward)
  m.def("set_predicted", [](int64_t device, int64_t P, int64_t W, int64_t H, int64_t num) {
    DeviceState& st = state_of((int)device);
    std::lock_guard<std::mutex> g(st.mu);
    st.predicted[std::make_tuple(P, W, H)] = (uint64_t)num;
  });
}
