// b2r_torch.cpp -- compiled torch binding of the eager drop-in path.
//
// `GaussianRasterizer.forward` (exavatar_release_b200/rasterizer.py; reference call site avatar/common/nets/module.py:632-640)
// spent ~0.2 ms of Python per render around ~0.1 ms of kernel launches: building ctypes structs, a dozen torch.empty calls,
// the autograd.Function trampolines in both directions (tools/eager_profile.py).  This file is the same
// host logic -- argument normalisation, the duplicate-capacity policy with its pinned-host status mirror, workspace
// allocation, the saved context, the backward call -- as a C++ torch::autograd::Function over the SAME C ABI
// (include/b200raster.h, libb200raster.so).  No kernels here and no second implementation of anything on the device.
//
// Scope: every rasteriser call -- adaptive capacity, fixed capacity (no polling, capturable in a CUDA graph) and
// debug=True (synchronises after each call).  rasterizer.py only maps the public arguments onto `rasterize` and dumps
// the inputs of a failed debug call.  Also here: the host side of optim.Adam's step (`adam_stage`, `adam_launch`), whose walk over
// thousands of SMPL-X param groups per step costs milliseconds in Python.
#include <torch/extension.h>

#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>
#include <cuda_runtime.h>

#include <chrono>
#include <cmath>
#include <cstring>
#include <deque>
#include <map>
#include <memory>
#include <mutex>
#include <stdexcept>
#include <string>
#include <tuple>
#include <vector>

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

// ctx buffers of the 64 most recent fixed-capacity calls: nothing is polled in that mode, so `overflowed()` reads their
// status blocks after the step.  Never destroyed, so no tensor is freed at exit after the CUDA allocator is gone.
struct RecentContexts {
  std::mutex mu;
  std::deque<at::Tensor> bufs;
};

RecentContexts& recent() {
  static RecentContexts* r = new RecentContexts();
  return *r;
}

// Library errors leave as std::runtime_error (RuntimeError in Python), not through TORCH_CHECK: on the H100 a c10::Error
// thrown here, with the call's CUDA buffers live, took the process down (SIGSEGV) instead of reaching the caller.
void check(int rc, const char* what) {
  if (rc != B2R_OK)
    throw std::runtime_error(std::string("b200raster: ") + what + " failed: " + b2r_strerror(rc) + " (cuda error " +
                             std::to_string(b2r_last_cuda_error()) + ")");
}

// debug=True (B2R_FLAG_DEBUG): wait for the call, so that a fault surfaces here rather than at a later API call
void sync_if_debug(uint32_t flags, cudaStream_t stream, const char* what) {
  if (!(flags & B2R_FLAG_DEBUG)) return;
  const cudaError_t e = cudaStreamSynchronize(stream);
  if (e != cudaSuccess)
    throw std::runtime_error(std::string("b200raster: ") + what + " failed on the device: " + cudaGetErrorString(e));
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
// The device tan(fov) pair: two contiguous fp32 values on the render's device.  Checked by shape only -- its values are
// never read on the host (the kernels cull everything when they are not finite and > 0).
at::Tensor device_tanfov(const at::Tensor& t, const c10::Device& dev) {
  TORCH_CHECK(t.is_cuda() && t.device() == dev, "b200raster: `tanfov` must be a CUDA tensor on the render's device");
  TORCH_CHECK(t.scalar_type() == at::kFloat && t.numel() == 2 && t.is_contiguous(),
              "b200raster: `tanfov` must be 2 contiguous float32 values");
  return t;
}
bool present(const c10::optional<at::Tensor>& t) { return t.has_value() && t->defined() && t->numel() > 0; }
const float* fptr(const at::Tensor& t) { return t.defined() && t.numel() > 0 ? t.data_ptr<float>() : nullptr; }

B2RScene make_scene(int64_t P, int64_t H, int64_t W, int64_t sh_degree, uint32_t flags, double scale_modifier, double tanfovx,
                    double tanfovy, const at::Tensor& bg, const at::Tensor& view, const at::Tensor& proj,
                    const at::Tensor& campos, const at::Tensor& means3D, const at::Tensor& shs, const at::Tensor& colors,
                    const at::Tensor& opac, const at::Tensor& scales, const at::Tensor& rots, const at::Tensor& cov,
                    const at::Tensor& tanfov) {
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
  sc.tanfov = fptr(tanfov);  // device tan(fov) (2), never read on the host; undefined: the floats above
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
                               const at::Tensor& campos_in, bool speculative, double headroom, int64_t fixed_capacity,
                               bool debug, const c10::optional<at::Tensor>& tanfov_in,
                               const c10::optional<at::Tensor>& status_out) {
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
      if (status_out.has_value() && status_out->defined()) status_out->zero_();  // no entries, no overflow
      ctx->mark_non_differentiable({radii});
      return {color, radii, depth, alpha};
    }
    const at::Tensor bg = f32c(bg_in.to(dev), "bg"), view = f32c(view_in.to(dev), "viewmatrix");
    const at::Tensor proj = f32c(proj_in.to(dev), "projmatrix"), campos = f32c(campos_in.to(dev), "campos");
    const at::Tensor tanfov = tanfov_in.has_value() && tanfov_in->defined() ? device_tanfov(*tanfov_in, dev) : at::Tensor();
    const bool want_status = status_out.has_value() && status_out->defined();
    if (want_status)
      TORCH_CHECK(status_out->is_cuda() && status_out->device() == dev && status_out->scalar_type() == at::kByte &&
                      status_out->is_contiguous() && (size_t)status_out->numel() == sizeof(B2RStatus),
                  "b200raster: `status` must be ", sizeof(B2RStatus), " contiguous uint8 bytes on the render's device");
    const uint32_t flags = debug ? B2R_FLAG_DEBUG : 0u;
    const B2RScene sc = make_scene(P, H, W, sh_degree, flags, scale_modifier, tanfovx, tanfovy, bg, view, proj, campos,
                                   means3D, shs, colors, opac, scales, rots, cov, tanfov);
    const size_t ctx_bytes = b2r_ctx_bytes((int32_t)P, (int32_t)W, (int32_t)H);
    at::Tensor ctx_buf = at::empty({(int64_t)ctx_bytes}, u8);
    B2RForwardOutputs out{color.data_ptr<float>(), depth.data_ptr<float>(), alpha.data_ptr<float>(), radii.data_ptr<int32_t>()};

    at::Tensor ids, ck;
    uint64_t cap = 0;
    auto workspace = [&](uint64_t capacity, uint64_t* mirror, uint64_t token) {
      cap = capacity;
      ids = at::empty({(int64_t)std::max<uint64_t>(cap, 1)}, i32);
      const size_t sbytes = b2r_scratch_bytes((int32_t)P, (int32_t)W, (int32_t)H, cap);
      at::Tensor scratch = at::empty({(int64_t)sbytes}, u8);  // recycled by the caching allocator in stream order
      size_t ckb = 0;
      ck = at::Tensor();
      if (need_grad) {  // segment table + blend-state checkpoints: the backward replays list segments independently
        ckb = b2r_checkpoint_bytes((int32_t)W, (int32_t)H, cap);
        ck = at::empty({(int64_t)ckb}, u8);
      }
      B2RWorkspace ws{ctx_buf.data_ptr(), ctx_bytes, (uint32_t*)ids.data_ptr<int32_t>(), cap, scratch.data_ptr(), sbytes,
                      mirror, token, ck.defined() ? ck.data_ptr() : nullptr, ckb};
      return ws;
    };
    if (fixed_capacity >= 0) {
      // no pinned allocation (state_of), lock or poll: the call is capturable in a CUDA graph.  An overflow truncates
      // the lists (never corrupts them) and is reported by `overflowed()` from the status block.
      const B2RWorkspace ws = workspace((uint64_t)fixed_capacity, nullptr, 0);
      check(b2r_forward(&sc, &ws, &out, stream), "b2r_forward");
      RecentContexts& r = recent();
      std::lock_guard<std::mutex> g(r.mu);
      r.bufs.push_back(ctx_buf);
      if (r.bufs.size() > 64) r.bufs.pop_front();
    } else {
      DeviceState& st = state_of(dev.index());
      uint64_t* mirror = const_cast<uint64_t*>(st.mirror);
      std::lock_guard<std::mutex> g(st.mu);
      const auto key = std::make_tuple(P, W, H);
      const auto it = st.predicted.find(key);
      uint64_t num = 0;
      if (speculative && it != st.predicted.end()) {
        uint64_t token = ++st.token;
        B2RWorkspace ws = workspace((uint64_t)((double)it->second * headroom) + 4096, mirror, token);
        check(b2r_forward(&sc, &ws, &out, stream), "b2r_forward");
        num = wait_mirror(st, token, stream);
        if (num > cap) {  // misprediction: the whole forward again with the exact size
          token = ++st.token;
          ws = workspace(num, mirror, token);
          check(b2r_forward(&sc, &ws, &out, stream), "b2r_forward");
          num = wait_mirror(st, token, stream);
        }
      } else {
        const uint64_t token = ++st.token;
        B2RWorkspace ws0{ctx_buf.data_ptr(), ctx_bytes, nullptr, 0, nullptr, 0, mirror, token, nullptr, 0};
        check(b2r_forward_project(&sc, &ws0, radii.data_ptr<int32_t>(), stream), "b2r_forward_project");
        num = wait_mirror(st, token, stream);
        B2RWorkspace ws = workspace(num, mirror, token);
        check(b2r_forward_render(&sc, &ws, &out, stream), "b2r_forward_render");
      }
      st.predicted[key] = num;
    }
    // this call's own status block, copied in stream order (a graph node when captured): no host read, no shared state
    if (want_status)
      TORCH_CHECK(cudaMemcpyAsync(status_out->data_ptr(), ctx_buf.data_ptr(), sizeof(B2RStatus), cudaMemcpyDeviceToDevice,
                                  stream) == cudaSuccess, "b200raster: cannot copy the status block");
    sync_if_debug(flags, stream, "b2r_forward");
    // what must survive until backward (SURVEY.md section 8b "Ownership"); undefined tensors are saved as such
    ctx->save_for_backward({means3D, shs, colors, opac, scales, rots, cov, bg, view, proj, campos, ctx_buf, ids, ck, tanfov});
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
    // one entry per forward argument: 8 tensors, then 15 settings and the status output
    variable_list out(24);
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
                     &ids = sv[12], &ck = sv[13], &tanfov = sv[14];
    const int64_t H = ctx->saved_data["H"].toInt(), W = ctx->saved_data["W"].toInt();
    const auto dev = means3D.device();
    c10::cuda::CUDAGuard guard(dev);
    const cudaStream_t stream = c10::cuda::getCurrentCUDAStream(dev.index()).stream();
    const B2RScene sc = make_scene(P, H, W, ctx->saved_data["sh_degree"].toInt(), (uint32_t)ctx->saved_data["flags"].toInt(),
                                   ctx->saved_data["scale_modifier"].toDouble(), ctx->saved_data["tanfovx"].toDouble(),
                                   ctx->saved_data["tanfovy"].toDouble(), bg, view, proj, campos, means3D, shs, colors, opac,
                                   scales, rots, cov, tanfov);
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
    sync_if_debug(sc.flags, stream, "b2r_backward");
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
                                  int64_t sh_degree, const at::Tensor& campos, bool speculative, double headroom,
                                  int64_t fixed_capacity, bool debug, const c10::optional<at::Tensor>& tanfov,
                                  const c10::optional<at::Tensor>& status) {
  return RasterizeFn::apply(means3D, means2D, sh, colors, opac, scales, rots, cov, H, W, tanfovx, tanfovy, bg, scale_modifier,
                            view, proj, sh_degree, campos, speculative, headroom, fixed_capacity, debug, tanfov, status);
}

// ---- optim.Adam's step: the walk over the param groups, the state, the scalars and the segment table ----------------

// torch/optim/adam.py _multi_tensor_adam (capturable=False): the Python float expressions, in double (Python's `**` is
// C pow), rounded to fp32 once by the foreach ops' scalar arguments.
void adam_scalars(double lr, double beta1, double beta2, double eps, double step, B2RAdamSegment& s) {
  const double bc1 = 1 - std::pow(beta1, step);
  const double bc2 = 1 - std::pow(beta2, step);
  s.lerp_weight = (float)(1 - beta1);
  s.beta2 = (float)beta2;
  s.one_minus_beta2 = (float)(1 - beta2);
  s.bc2_sqrt = (float)std::pow(bc2, 0.5);
  s.eps = (float)eps;
  s.step_size = (float)((lr / bc1) * -1);
}

// The param as rows of row_len contiguous floats, row_stride apart: a contiguous tensor, or a view such as ExAvatar's
// feature_dc = feature[:, 0:1, :] of a (P,16,3) tensor.  False for any other layout.
bool row_layout(const at::Tensor& p, int64_t& row_len, int64_t& row_stride) {
  const auto sz = p.sizes(), st = p.strides();
  int i = (int)sz.size() - 1;
  row_len = 1;
  for (; i >= 0 && (sz[i] == 1 || st[i] == row_len); i--) row_len *= sz[i];
  row_stride = row_len;
  int64_t span = -1;
  for (; i >= 0; i--) {
    if (sz[i] == 1) continue;
    if (span < 0) {
      row_stride = st[i];
    } else if (st[i] != span) {
      return false;
    }
    span = st[i] * sz[i];
  }
  return row_stride >= row_len;
}

[[noreturn]] void value_error(const std::string& what) { throw py::value_error("Adam: " + what); }

// The host half of an Adam step over every param with a gradient in `groups` (the optimizer's param_groups), with
// torch.optim.Adam's lazy state in `state`: the walk, the lazy state, the step counts, the scalars and the segment
// table, written into the resident device table `table` (reallocated when undefined or too small) with one async H2D
// copy from pinned memory on the current stream of `device`.  A group with a true "frame_rows" key has dim 0 = frame:
// only row `rows` of each of its params is stepped, with that row's own count in state["step"], a (rows,) CPU float32
// tensor.  Returns (table, n_segments, n_chunks, layout): `layout` names what a launch captured in a graph depends on
// (the tensors and their sizes, the chunk count; not the rows, the scalars or the counts).  Every check runs before
// anything is created or counted.  When `expect` is not None and the layout differs from it, no state is created,
// nothing is counted, copied or written, and the table comes back as it was.  With no gradient at all the table also
// comes back as it was (undefined if it never existed) and n_chunks is 0: nothing to launch.
py::tuple adam_stage(const py::list& groups, const py::object& state, int64_t device, int64_t chunk,
                     const py::object& rows, const c10::optional<at::Tensor>& table_in, const py::object& expect) {
  at::Tensor table = table_in.has_value() ? *table_in : at::Tensor();
  const at::Device dev(at::kCUDA, (c10::DeviceIndex)device);
  struct Entry {
    py::handle ph;
    at::Tensor p, g;
    bool frame_rows;
    int64_t row;  // -1: the whole tensor
    int64_t numel, row_len, row_stride;
    double lr, beta1, beta2, eps;
  };
  // pass 1: every check, nothing created or counted
  std::vector<Entry> entries;
  for (const py::handle gh : groups) {
    const py::dict group = py::reinterpret_borrow<py::dict>(gh);
    const bool frame_rows = group.contains("frame_rows") && py::bool_(group["frame_rows"]);
    bool scalars = false;
    double lr = 0, beta1 = 0, beta2 = 0, eps = 0;
    for (const py::handle ph : py::reinterpret_borrow<py::list>(group["params"])) {
      const at::Tensor p = ph.cast<at::Tensor>();
      const at::Tensor& g = p.grad();
      if (!g.defined()) continue;
      if (g.is_sparse()) value_error("sparse gradients are not supported");
      int64_t row = -1;
      if (frame_rows) {
        if (rows.is_none()) value_error("a frame-row group is stepped only with `rows` (the frame's slot)");
        if (p.dim() < 1 || !p.is_contiguous()) value_error("a frame-row parameter must be contiguous with dim 0 = frame");
        row = rows.cast<int64_t>();
        if (row < 0 || row >= p.size(0))
          value_error("rows=" + std::to_string(row) + " lies outside a frame-row parameter's " +
                      std::to_string(p.size(0)) + " rows");
      }
      if (p.device() != dev || p.scalar_type() != at::kFloat)
        value_error("parameters must be float32 tensors on the optimizer's CUDA device");
      if (g.scalar_type() != at::kFloat || g.device() != dev || g.sizes() != p.sizes() || !g.is_contiguous())
        value_error("a gradient must be a contiguous float32 tensor shaped and placed as its parameter");
      if (!scalars) {
        lr = group["lr"].cast<double>();
        const py::tuple betas = group["betas"];
        beta1 = betas[0].cast<double>();
        beta2 = betas[1].cast<double>();
        eps = group["eps"].cast<double>();
        scalars = true;
      }
      if (state.contains(ph)) {
        const py::object st = state[ph];
        if (py::len(st) != 0) {
          const at::Tensor step = st["step"].cast<at::Tensor>();
          const at::Tensor m = st["exp_avg"].cast<at::Tensor>(), v = st["exp_avg_sq"].cast<at::Tensor>();
          if (!step.device().is_cpu() || step.scalar_type() != at::kFloat || !step.is_contiguous() ||
              (frame_rows ? step.dim() != 1 || step.size(0) != p.size(0) : step.numel() != 1))
            value_error(frame_rows ? "state 'step' of a frame-row parameter must be a (rows,) CPU float32 tensor"
                                   : "state 'step' must be a CPU float32 scalar tensor");
          for (const at::Tensor* t : {&m, &v})
            if (t->device() != dev || t->scalar_type() != at::kFloat || t->sizes() != p.sizes() || !t->is_contiguous())
              value_error("exp_avg / exp_avg_sq must be contiguous float32 tensors shaped and placed as their parameter");
        }
      }
      const int64_t numel = row < 0 ? p.numel() : p.numel() / p.size(0);
      int64_t row_len = numel, row_stride = numel;
      if (numel > 0 && row < 0 && !row_layout(p, row_len, row_stride))
        value_error("a parameter must be contiguous or rows of contiguous floats at one stride");
      entries.push_back({ph, p, g, frame_rows, row, numel, row_len, row_stride, lr, beta1, beta2, eps});
    }
  }
  int64_t n_chunks = 0;
  for (const Entry& e : entries)
    if (e.numel > 0) n_chunks += (e.numel + chunk - 1) / chunk;
  // the layout a captured launch depends on; moments not created yet count as address 0
  auto layout_of = [&](const std::vector<std::pair<const void*, const void*>>& moments) {
    std::vector<int64_t> layout;
    for (size_t i = 0; i < entries.size(); ++i) {
      const Entry& e = entries[i];
      for (const int64_t x : {(int64_t)(uintptr_t)e.p.data_ptr(), (int64_t)(uintptr_t)e.g.data_ptr(),
                              (int64_t)(uintptr_t)moments[i].first, (int64_t)(uintptr_t)moments[i].second, e.numel,
                              e.row_len, e.row_stride, (int64_t)(e.row >= 0)})
        layout.push_back(x);
    }
    layout.push_back(n_chunks);
    return py::bytes(reinterpret_cast<const char*>(layout.data()), layout.size() * sizeof(int64_t));
  };
  std::vector<std::pair<const void*, const void*>> moments;
  for (const Entry& e : entries) {
    const void *m = nullptr, *v = nullptr;
    if (state.contains(e.ph) && py::len(state[e.ph]) != 0) {
      m = state[e.ph]["exp_avg"].cast<at::Tensor>().data_ptr();
      v = state[e.ph]["exp_avg_sq"].cast<at::Tensor>().data_ptr();
    }
    moments.emplace_back(m, v);
  }
  if (!expect.is_none() && !layout_of(moments).equal(expect))
    return py::make_tuple(table, 0, 0, layout_of(moments));
  // pass 2: lazy state, counts, scalars, segments
  std::vector<B2RAdamSegment> segs;
  moments.clear();
  n_chunks = 0;
  for (const Entry& e : entries) {
    py::object st = state[e.ph];  // a defaultdict: the first access creates the empty state
    if (py::len(st) == 0) {       // torch.optim.Adam._init_group's lazy state (capturable=False, fused=False)
      st["step"] = e.frame_rows ? at::zeros({e.p.size(0)}, at::TensorOptions().dtype(at::kFloat))
                                : at::zeros({}, at::TensorOptions().dtype(at::kFloat));
      st["exp_avg"] = at::zeros_like(e.p, at::MemoryFormat::Preserve);
      st["exp_avg_sq"] = at::zeros_like(e.p, at::MemoryFormat::Preserve);
    }
    const at::Tensor step = st["step"].cast<at::Tensor>();
    const at::Tensor m = st["exp_avg"].cast<at::Tensor>(), v = st["exp_avg_sq"].cast<at::Tensor>();
    moments.emplace_back(m.data_ptr(), v.data_ptr());
    // as torch's _foreach_add_(steps, tensor(1.), alpha=1.): every step count of a param with a gradient advances
    float* sp = step.data_ptr<float>() + (e.row < 0 ? 0 : e.row);
    *sp = *sp + 1.0f;
    if (e.numel == 0) continue;
    const int64_t off = e.row < 0 ? 0 : e.row * e.numel;
    B2RAdamSegment s{};
    s.row_len = e.row_len;
    s.row_stride = e.row_stride;
    s.param = e.p.data_ptr<float>() + off;
    s.grad = e.g.data_ptr<float>() + off;
    s.exp_avg = m.data_ptr<float>() + off;
    s.exp_avg_sq = v.data_ptr<float>() + off;
    s.numel = e.numel;
    s.first_chunk = n_chunks;
    n_chunks += (e.numel + chunk - 1) / chunk;
    adam_scalars(e.lr, e.beta1, e.beta2, e.eps, (double)*sp, s);
    segs.push_back(s);
  }
  const py::bytes layout = layout_of(moments);
  if (entries.empty()) return py::make_tuple(table, 0, 0, layout);
  const int64_t bytes = (int64_t)(segs.size() * sizeof(B2RAdamSegment));
  c10::cuda::CUDAGuard guard(dev);
  if (!table.defined() || table.device() != dev || table.numel() < std::max<int64_t>(bytes, 1))
    table = at::empty({std::max<int64_t>(bytes, 1)}, at::TensorOptions().dtype(at::kByte).device(dev));
  if (bytes > 0) {
    // the caching host allocator records the copy on the stream and keeps `host` from reuse until the copy has run
    at::Tensor host = at::empty({bytes}, at::TensorOptions().dtype(at::kByte).pinned_memory(true));
    std::memcpy(host.data_ptr(), segs.data(), (size_t)bytes);
    table.narrow(0, 0, bytes).copy_(host, /*non_blocking=*/true);
  }
  return py::make_tuple(table, (int64_t)segs.size(), n_chunks, layout);
}

// The device half: one launch of csrc/adam.cu over a staged table on the current stream of `device` (capturable)
void adam_launch(const at::Tensor& table, int64_t n_segments, int64_t n_chunks, int64_t device) {
  if (n_chunks == 0) return;
  c10::cuda::CUDAGuard guard((c10::DeviceIndex)device);
  const cudaStream_t stream = c10::cuda::getCurrentCUDAStream((c10::DeviceIndex)device).stream();
  check(b2r_adam_step((const B2RAdamSegment*)table.data_ptr(), (int32_t)n_segments, n_chunks, stream), "b2r_adam_step");
}

}  // namespace

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.def("adam_stage", &adam_stage, "optim.Adam.stage: the host half of a step, staged into a resident device table");
  m.def("adam_launch", &adam_launch, "optim.Adam.launch: one launch of csrc/adam.cu over a staged table");
  m.def("adam_scalars", [](double lr, double beta1, double beta2, double eps, double step) {
    B2RAdamSegment s{};
    adam_scalars(lr, beta1, beta2, eps, step, s);
    return std::vector<float>{s.lerp_weight, s.beta2, s.one_minus_beta2, s.bc2_sqrt, s.eps, s.step_size};
  }, "the fp32 scalars of one tensor's step: (lerp_weight, beta2, one_minus_beta2, bc2_sqrt, eps, step_size)");
  m.def("adam_row_layout", [](const at::Tensor& p) {
    int64_t row_len = 0, row_stride = 0;
    const bool ok = row_layout(p, row_len, row_stride);
    return std::make_tuple(ok, row_len, row_stride);
  }, "(representable, row_len, row_stride) of a param for the Adam step");
  m.def("rasterize", &rasterize, "GaussianRasterizer forward with autograd (compiled host path over libb200raster.so); "
        "fixed_capacity < 0: adaptive duplicate capacity; tanfov: (2) device tan(fov) in place of tanfovx / tanfovy; "
        "status: a B2RStatus-sized uint8 CUDA tensor that receives this call's status block, in stream order",
        py::arg("means3D"), py::arg("means2D"), py::arg("sh"), py::arg("colors"), py::arg("opac"), py::arg("scales"),
        py::arg("rots"), py::arg("cov"), py::arg("H"), py::arg("W"), py::arg("tanfovx"), py::arg("tanfovy"), py::arg("bg"),
        py::arg("scale_modifier"), py::arg("view"), py::arg("proj"), py::arg("sh_degree"), py::arg("campos"),
        py::arg("speculative"), py::arg("headroom"), py::arg("fixed_capacity"), py::arg("debug"),
        py::arg("tanfov") = py::none(), py::arg("status") = py::none());
  m.def("abi_version", []() { return b2r_abi_version(); });
  m.def("recent_contexts", []() {  // ctx buffers of the recent fixed-capacity calls, oldest first
    RecentContexts& r = recent();
    std::lock_guard<std::mutex> g(r.mu);
    return std::vector<at::Tensor>(r.bufs.begin(), r.bufs.end());
  });
  m.def("clear_recent", []() {
    RecentContexts& r = recent();
    std::lock_guard<std::mutex> g(r.mu);
    r.bufs.clear();
  });
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
