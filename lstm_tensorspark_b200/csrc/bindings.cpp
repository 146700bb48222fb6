// Python bindings for the sm_90a kernels (the only translation unit that sees torch headers).
// Every function validates device / dtype / contiguity, takes the CURRENT torch CUDA stream (so the kernels
// are stream-ordered with the rest of the step and capturable in CUDA graphs) and forwards raw pointers to the
// C-ABI launchers defined next to the kernels.
#include <torch/extension.h>
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAException.h>
#include <cuda_runtime.h>

#include <optional>
#include <string>
#include <vector>

using torch::Tensor;

extern "C" {
int ts_lstm_pointwise_fwd(const void*, const float*, const float*, void*, float*, void*, int, int, int, cudaStream_t, const void*,
                          const int*, int);
int ts_transpose01_rows(const void*, void*, int, int, long long, cudaStream_t);
int ts_lstm_seq_cluster_probe(int);
int ts_lstm_seq_config(int, int, int, int, int*);
int ts_transpose2d_b16(const void*, void*, int, int, cudaStream_t);
int ts_colsum_bf16(const void*, float*, void*, int, int, int, int, int, int, cudaStream_t);
long long ts_colsum_scratch_bytes(int, int);
int ts_lstm_pointwise_bwd(const void*, const float*, const float*, const void*, const float*, const float*, void*,
                          float*, int, int, int, cudaStream_t, const int*, int, float*);
int ts_xent_rows(const float*, const long long*, float*, float*, int*, int, int, cudaStream_t);
int ts_flat_adam(float*, const float*, float*, float*, void*, long long, float, float, float, float, float, float,
                 cudaStream_t, int*, long long);
int ts_flat_sgd(float*, const float*, void*, long long, float, float, float, cudaStream_t, long long);
int ts_cast_bf16(const float*, void*, long long, cudaStream_t);
int ts_fused_allreduce(const unsigned long long*, unsigned long long, unsigned long long, unsigned long long, float*,
                       float*, unsigned int*, int*, long long, int, int, int, int, int, int, float, float, float, float,
                       float, double, cudaStream_t, int*, long long, int, int);
int ts_ar_bump_step(int*, cudaStream_t);
int ts_ar_max_blocks();
int ts_ar_flag_words();
int ts_ar_slots();
int ts_head_fwd_tc(const void*, int, const float*, const float*, const long long*, float*, float*, float*, int*, int, int, int, cudaStream_t);
int ts_head_logits_generic(const void*, const float*, const float*, float*, int, int, int, int, cudaStream_t);
int ts_head_bwd(const void*, const float*, const float*, const float*, void*, float*, float*, int, int, int, int, int, cudaStream_t);
int ts_gemm_generic(const void*, const void*, void*, const float*, int, int, int, long long, long long, long long, long long, long long,
                    int, int, int, float, cudaStream_t);
int ts_gemm2(const void*, const void*, void*, const float*, int, int, int, int, int, int, int, int, int, int, int, int, int,
             const unsigned int*, const int*, unsigned int*, int*, int, int, int, int, cudaStream_t);
int ts_lstm_seq_fwd(const void*, const void*, const float*, const void*, const float*, void*, const float*, void*, void*, int,
                    int, int, unsigned int*, int, cudaStream_t, const void*, const unsigned int*, int, int, int, const int*, int,
                    void*, const int*, const unsigned int*);
int ts_lstm_seq_bwd(const void*, const void*, const void*, const float*, const void*, float*, float*, void*, void*, int,
                    int, int, unsigned int*, int, cudaStream_t, const unsigned int*, int, int, int, const int*, int,
                    const int*, const unsigned int*);
int ts_dropout(const void*, void*, int, int, int, int, int, const int*, const unsigned int*, cudaStream_t);
int ts_lstm_seq_prologue(const void*, const float*, void*, float*, void*, unsigned int*, int, int, cudaStream_t);
const char* ts_last_error();
}

namespace {

void check(int rc, const char* what) {
  if (rc != 0) {
    std::string msg = std::string(what) + " failed: rc=" + std::to_string(rc);
    if (rc > 0) msg += std::string(" (") + cudaGetErrorString((cudaError_t)rc) + ")";
    const char* le = ts_last_error();
    if (le && le[0]) msg += std::string(" [") + le + "]";
    TORCH_CHECK(false, msg);
  }
}
cudaStream_t stream() { return at::cuda::getCurrentCUDAStream().stream(); }
void chk_cuda(const Tensor& t, const char* n) {
  TORCH_CHECK(t.is_cuda(), n, " must be a CUDA tensor");
  TORCH_CHECK(t.is_contiguous(), n, " must be contiguous");
}
int is_bf16(const Tensor& t) {
  TORCH_CHECK(t.scalar_type() == torch::kBFloat16 || t.scalar_type() == torch::kFloat32, "dtype must be bf16 or fp32");
  return t.scalar_type() == torch::kBFloat16 ? 1 : 0;
}
const float* fptr(const std::optional<Tensor>& t) { return t.has_value() ? t->data_ptr<float>() : nullptr; }
// Per-row sequence lengths: int32 [B] on the batch's device.  The values (1 <= len <= T) are not checked here: that would
// need a device-to-host copy on every call.
const int* lengths_ptr(const std::optional<Tensor>& lengths, int64_t B, const Tensor& like) {
  if (!lengths.has_value()) return nullptr;
  const Tensor& l = *lengths;
  TORCH_CHECK(l.is_cuda() && l.device() == like.device(), "lengths must be on the batch's device");
  TORCH_CHECK(l.scalar_type() == torch::kInt32, "lengths must be int32");
  TORCH_CHECK(l.dim() == 1 && l.size(0) == B, "lengths must be [B] (B = ", B, ")");
  TORCH_CHECK(l.is_contiguous(), "lengths must be contiguous");
  return l.data_ptr<int>();
}
// Dropout between stacked layers (ts_common.cuh DropSpec): step = the device-resident int32 step counter [1] (None = no
// dropout), desc = {key0, key1, thr, c2, row0}.  -> counter pointer (null without dropout); desc is converted into `out`.
const int* drop_args(const std::optional<Tensor>& step, const std::vector<int64_t>& desc, const Tensor& like, unsigned int (&out)[5]) {
  if (!step.has_value()) return nullptr;
  TORCH_CHECK(step->is_cuda() && step->device() == like.device() && step->scalar_type() == torch::kInt32 && step->numel() == 1,
              "dropout: the step counter must be an int32 [1] tensor on the batch's device");
  TORCH_CHECK(desc.size() == 5, "dropout: desc = {key0, key1, thr, c2, row0}");
  TORCH_CHECK(desc[2] >= 1 && desc[2] <= 65535 && desc[4] >= 0, "dropout: thr in [1, 65535], row0 >= 0");
  for (int i = 0; i < 5; ++i) out[i] = (unsigned int)(uint32_t)desc[i];
  return step->data_ptr<int>();
}

// Direction of a persistent-kernel launch: reverse = the reverse-time half of a bidirectional layer (h_seq / c_seq row T holds
// the initial state).  The layer wavefront's dataflow gating (in_gate / extra_signal) is forward-only.
int direction_flag(bool reverse, const std::optional<Tensor>& in_gate, bool extra_signal) {
  TORCH_CHECK(!reverse || (!in_gate.has_value() && !extra_signal), "reverse: the layer wavefront (in_gate / extra_signal) is forward-only");
  return reverse ? 1 : 0;
}

// x [B,T,D] contiguous -> [T,B,D] contiguous (row permutation at copy speed)
Tensor transpose01(const Tensor& x) {
  chk_cuda(x, "x");
  TORCH_CHECK(x.dim() == 3 && x.is_contiguous(), "transpose01: expected a contiguous [B,T,D] tensor");
  c10::cuda::CUDAGuard g(x.device());
  const int B = x.size(0), T = x.size(1);
  const long long row_bytes = (long long)x.size(2) * x.element_size();
  TORCH_CHECK(row_bytes % 16 == 0, "transpose01: row size must be a multiple of 16 bytes");
  auto out = torch::empty({x.size(1), x.size(0), x.size(2)}, x.options());
  check(ts_transpose01_rows(x.data_ptr(), out.data_ptr(), B, T, row_bytes, stream()), "transpose01");
  return out;
}

// [R,C] bf16/fp16 contiguous -> [C,R] contiguous (shared-memory tile transpose)
Tensor transpose2d(const Tensor& x) {
  chk_cuda(x, "x");
  TORCH_CHECK(x.dim() == 2 && x.is_contiguous() && x.element_size() == 2, "transpose2d: expected a contiguous 2-D 16-bit tensor");
  c10::cuda::CUDAGuard g(x.device());
  auto out = torch::empty({x.size(1), x.size(0)}, x.options());
  check(ts_transpose2d_b16(x.data_ptr(), out.data_ptr(), (int)x.size(0), (int)x.size(1), stream()), "transpose2d");
  return out;
}

// per-device scratch of the deterministic column-sum kernel (slab partials + tickets; the kernel leaves the tickets zero)
void* colsum_scratch(const Tensor& x) {
  static std::vector<Tensor> bufs(64);
  const int dev = x.device().index();
  const int64_t need = ts_colsum_scratch_bytes((int)x.size(0), (int)x.size(1));
  if (!bufs[dev].defined() || bufs[dev].numel() < need)        // (a bigger buffer starts with zeroed tickets again)
    bufs[dev] = torch::zeros({need}, torch::TensorOptions().device(x.device()).dtype(torch::kUInt8));
  return bufs[dev].data_ptr();
}

// column sums of a contiguous bf16 [rows, cols] matrix -> fp32 [cols]
Tensor colsum_bf16(const Tensor& x) {
  chk_cuda(x, "x");
  TORCH_CHECK(x.dim() == 2 && x.is_contiguous() && is_bf16(x) && x.size(1) % 256 == 0, "colsum_bf16: contiguous bf16 [rows, cols], cols % 256 == 0");
  c10::cuda::CUDAGuard g(x.device());
  auto out = torch::empty({x.size(1)}, x.options().dtype(torch::kFloat32));
  check(ts_colsum_bf16(x.data_ptr(), out.data_ptr<float>(), colsum_scratch(x), (int)x.size(0), (int)x.size(1), (int)x.size(1), 0, 0, 0, stream()), "colsum_bf16");
  return out;
}

// column sums written (overwrite) or accumulated into an existing fp32 [cols] tensor; pdl: launch as a programmatic dependent of
// the previous kernel of the stream (a weight-gradient GEMM that reads the same matrix and leaves SMs idle); max_ctas > 0 caps
// the grid (the same sums, computed by fewer CTAs)
void colsum_bf16_into(const Tensor& x, Tensor out, bool overwrite, bool pdl, int64_t col0, int64_t ncols, int64_t max_ctas) {
  chk_cuda(x, "x"); chk_cuda(out, "out");
  TORCH_CHECK(x.dim() == 2 && is_bf16(x) && x.size(1) % 256 == 0 && out.scalar_type() == torch::kFloat32 && out.numel() == x.size(1),
              "colsum_bf16_into: bf16 [rows, cols % 256 == 0] -> fp32 [cols]");
  if (ncols <= 0) { col0 = 0; ncols = x.size(1); }
  TORCH_CHECK(col0 % 256 == 0 && ncols % 256 == 0 && col0 + ncols <= x.size(1), "colsum_bf16_into: 256-aligned column range");
  c10::cuda::CUDAGuard g(x.device());
  check(ts_colsum_bf16((const char*)x.data_ptr() + 2 * col0, out.data_ptr<float>() + col0, colsum_scratch(x), (int)x.size(0), (int)ncols,
                       (int)x.size(1), overwrite ? 0 : 1, pdl ? 1 : 0, (int)max_ctas, stream()), "colsum_bf16_into");
}

// ---- generic LSTM cell epilogue -------------------------------------------------------------------------
// lengths (optional, with the step index t and h_prev [B,H] of pre's dtype): rows with t >= lengths[b] carry (h_prev, c_prev)
std::vector<Tensor> lstm_pointwise_fwd(const Tensor& pre, const Tensor& bias, const Tensor& c_prev, const std::optional<Tensor>& h_prev,
                                       const std::optional<Tensor>& lengths, int64_t t) {
  chk_cuda(pre, "pre"); chk_cuda(bias, "bias"); chk_cuda(c_prev, "c_prev");
  c10::cuda::CUDAGuard g(pre.device());
  int B = pre.size(0), H = pre.size(1) / 4;
  TORCH_CHECK(bias.scalar_type() == torch::kFloat32 && c_prev.scalar_type() == torch::kFloat32, "bias/c must be fp32");
  TORCH_CHECK(c_prev.numel() == (int64_t)B * H && bias.numel() == 4 * H, "shape mismatch");
  const int* lp = lengths_ptr(lengths, B, pre);
  if (lp) {
    TORCH_CHECK(h_prev.has_value(), "lstm_pointwise_fwd: lengths need h_prev");
    chk_cuda(*h_prev, "h_prev");
    TORCH_CHECK(h_prev->scalar_type() == pre.scalar_type() && h_prev->numel() == (int64_t)B * H, "h_prev: [B,H] in pre's dtype");
  }
  auto h = torch::empty({B, H}, pre.options());
  auto c = torch::empty({B, H}, c_prev.options());
  auto act = torch::empty_like(pre);
  check(ts_lstm_pointwise_fwd(pre.data_ptr(), bias.data_ptr<float>(), c_prev.data_ptr<float>(), h.data_ptr(),
                              c.data_ptr<float>(), act.data_ptr(), B, H, is_bf16(pre), stream(), lp ? h_prev->data_ptr() : nullptr,
                              lp, (int)t), "lstm_pointwise_fwd");
  return {h, c, act};
}

std::vector<Tensor> lstm_pointwise_bwd(const std::optional<Tensor>& dh_a, const std::optional<Tensor>& dh_b,
                                       const std::optional<Tensor>& dc_in, const Tensor& act, const Tensor& c_prev,
                                       const Tensor& c_new, const std::optional<Tensor>& lengths, int64_t t) {
  chk_cuda(act, "act"); chk_cuda(c_prev, "c_prev"); chk_cuda(c_new, "c_new");
  c10::cuda::CUDAGuard g(act.device());
  int B = act.size(0), H = act.size(1) / 4;
  const int* lp = lengths_ptr(lengths, B, act);
  if (dh_a.has_value()) { chk_cuda(*dh_a, "dh_a"); TORCH_CHECK(dh_a->scalar_type() == act.scalar_type(), "dh_a dtype"); }
  if (dh_b.has_value()) { chk_cuda(*dh_b, "dh_b"); TORCH_CHECK(dh_b->scalar_type() == torch::kFloat32, "dh_b fp32"); }
  if (dc_in.has_value()) { chk_cuda(*dc_in, "dc_in"); TORCH_CHECK(dc_in->scalar_type() == torch::kFloat32, "dc fp32"); }
  auto dpre = torch::empty_like(act);
  auto dc = torch::empty_like(c_prev);
  // with lengths: a third output, the dh handed straight to step t-1 (the total dh of padded rows, 0 elsewhere)
  Tensor dh_out = lp ? torch::empty_like(c_prev) : Tensor();
  check(ts_lstm_pointwise_bwd(dh_a.has_value() ? dh_a->data_ptr() : nullptr, fptr(dh_b), fptr(dc_in), act.data_ptr(),
                              c_prev.data_ptr<float>(), c_new.data_ptr<float>(), dpre.data_ptr(), dc.data_ptr<float>(),
                              B, H, is_bf16(act), stream(), lp, (int)t, lp ? dh_out.data_ptr<float>() : nullptr), "lstm_pointwise_bwd");
  if (lp) return {dpre, dc, dh_out};
  return {dpre, dc};
}

// x [..., B, H] (bf16 / fp32, contiguous; the leading dims are time steps t0, t0 + 1, ...) -> x * mask * scale (same dtype):
// the dropout of the generic path and of the one-step path, forward (x = h) and backward (x = the gradient).
Tensor dropout(const Tensor& x, const Tensor& step, const std::vector<int64_t>& desc, int64_t t0) {
  chk_cuda(x, "x");
  TORCH_CHECK(x.dim() >= 2, "dropout: x must be [..., B, H]");
  c10::cuda::CUDAGuard g(x.device());
  unsigned int dd[5];
  const int* ds = drop_args(step, desc, x, dd);
  const int64_t B = x.size(-2), H = x.size(-1), steps = B * H ? x.numel() / (B * H) : 0;
  auto y = torch::empty_like(x);
  check(ts_dropout(x.data_ptr(), y.data_ptr(), (int)steps, (int)B, (int)H, (int)t0, is_bf16(x), ds, dd, stream()), "dropout");
  return y;
}

// ---- head ---------------------------------------------------------------------------------------------------
std::vector<Tensor> xent_rows(const Tensor& logits, const Tensor& labels) {
  chk_cuda(logits, "logits"); chk_cuda(labels, "labels");
  c10::cuda::CUDAGuard g(logits.device());
  TORCH_CHECK(logits.scalar_type() == torch::kFloat32 && labels.scalar_type() == torch::kInt64, "dtypes");
  int B = logits.size(0), C = logits.size(1);
  auto dlogits = torch::empty_like(logits);
  auto loss = torch::zeros({1}, logits.options());
  auto correct = torch::zeros({1}, logits.options().dtype(torch::kInt32));
  check(ts_xent_rows(logits.data_ptr<float>(), (const long long*)labels.data_ptr<int64_t>(), dlogits.data_ptr<float>(),
                     loss.data_ptr<float>(), correct.data_ptr<int>(), B, C, stream()), "xent_rows");
  return {dlogits, loss, correct};
}

// Tensor-core head (csrc/head_wgmma.cu): bf16 h [B,H] (row pitch = stride(0)), fp32 W [H,C] / bias [C] -> logits, dlogits, loss sum,
// correct count.  Shapes the wgmma kernel does not take (fp32 h, C > 256, weight image > smem) run head_logits_generic +
// xent_rows - our own kernels, never a library GEMM.
std::vector<Tensor> head_fwd(const Tensor& h, const Tensor& W, const Tensor& bias, const Tensor& labels) {
  TORCH_CHECK(h.is_cuda() && h.dim() == 2 && h.stride(1) == 1, "head_fwd: h [B,H] with unit inner stride");
  chk_cuda(W, "W"); chk_cuda(bias, "bias"); chk_cuda(labels, "labels");
  c10::cuda::CUDAGuard g(h.device());
  const int B = h.size(0), H = h.size(1), C = W.size(1);
  TORCH_CHECK(W.size(0) == H && W.scalar_type() == torch::kFloat32 && bias.scalar_type() == torch::kFloat32, "head W/b");
  TORCH_CHECK(labels.scalar_type() == torch::kInt64 && labels.numel() == B, "labels int64 [B]");
  auto fo = torch::TensorOptions().device(h.device()).dtype(torch::kFloat32);
  auto logits = torch::empty({B, C}, fo), dlogits = torch::empty({B, C}, fo);
  auto loss = torch::zeros({1}, fo);
  auto correct = torch::zeros({1}, fo.dtype(torch::kInt32));
  int rc = -1;
  if (h.scalar_type() == torch::kBFloat16)
    rc = ts_head_fwd_tc(h.data_ptr(), (int)h.stride(0), W.data_ptr<float>(), bias.data_ptr<float>(), (const long long*)labels.data_ptr<int64_t>(),
                        logits.data_ptr<float>(), dlogits.data_ptr<float>(), loss.data_ptr<float>(), correct.data_ptr<int>(), B, H, C, stream());
  if (rc == -1) {
    auto hc = h.contiguous();
    check(ts_head_logits_generic(hc.data_ptr(), W.data_ptr<float>(), bias.data_ptr<float>(), logits.data_ptr<float>(), B, H, C, is_bf16(hc), stream()),
          "head_logits_generic");
    check(ts_xent_rows(logits.data_ptr<float>(), (const long long*)labels.data_ptr<int64_t>(), dlogits.data_ptr<float>(),
                       loss.data_ptr<float>(), correct.data_ptr<int>(), B, C, stream()), "xent_rows");
  } else {
    check(rc, "head_fwd_tc");
  }
  return {logits, dlogits, loss, correct};
}

// dh = (dloss * dlogits) W^T [B,H] (dtype of h), dW (+)= h^T (dloss * dlogits) [H,C], db (+)= column sums: one launch.
Tensor head_bwd(const Tensor& h, const Tensor& W, const Tensor& dlogits, const std::optional<Tensor>& dloss, Tensor dW, Tensor db,
                bool accumulate) {
  chk_cuda(h, "h"); chk_cuda(W, "W"); chk_cuda(dlogits, "dlogits"); chk_cuda(dW, "dW"); chk_cuda(db, "db");
  c10::cuda::CUDAGuard g(h.device());
  const int B = h.size(0), H = h.size(1), C = W.size(1);
  TORCH_CHECK(dW.scalar_type() == torch::kFloat32 && db.scalar_type() == torch::kFloat32 && dW.numel() == (int64_t)H * C && db.numel() == C, "head_bwd: dW/db");
  TORCH_CHECK(dlogits.scalar_type() == torch::kFloat32 && dlogits.numel() == (int64_t)B * C, "head_bwd: dlogits fp32 [B,C]");
  auto dh = torch::empty_like(h);
  check(ts_head_bwd(h.data_ptr(), W.data_ptr<float>(), dlogits.data_ptr<float>(), fptr(dloss), dh.data_ptr(), dW.data_ptr<float>(),
                    db.data_ptr<float>(), B, H, C, is_bf16(h), accumulate ? 1 : 0, stream()), "head_bwd");
  return dh;
}

// ---- optimizer ----------------------------------------------------------------------------------------------
void flat_adam(Tensor p, const Tensor& g, Tensor m, Tensor v, std::optional<Tensor> shadow, double lr_t, double b1,
               double b2, double eps, double wd, double gscale, std::optional<Tensor> step_dev, int64_t wd_numel) {
  chk_cuda(p, "p"); chk_cuda(g, "g"); chk_cuda(m, "m"); chk_cuda(v, "v");
  c10::cuda::CUDAGuard gd(p.device());
  TORCH_CHECK(p.numel() == g.numel() && p.numel() == m.numel() && p.numel() == v.numel(), "numel mismatch");
  check(ts_flat_adam(p.data_ptr<float>(), g.data_ptr<float>(), m.data_ptr<float>(), v.data_ptr<float>(),
                     shadow.has_value() ? shadow->data_ptr() : nullptr, p.numel(), lr_t, b1, b2, eps, wd, gscale, stream(),
                     step_dev.has_value() ? step_dev->data_ptr<int>() : nullptr, (long long)wd_numel),
        "flat_adam");
}
void flat_sgd(Tensor p, const Tensor& g, std::optional<Tensor> shadow, double lr, double wd, double gscale, int64_t wd_numel) {
  chk_cuda(p, "p"); chk_cuda(g, "g");
  c10::cuda::CUDAGuard gd(p.device());
  check(ts_flat_sgd(p.data_ptr<float>(), g.data_ptr<float>(), shadow.has_value() ? shadow->data_ptr() : nullptr,
                    p.numel(), lr, wd, gscale, stream(), (long long)wd_numel), "flat_sgd");
}
void cast_bf16(const Tensor& p, Tensor shadow) {
  chk_cuda(p, "p"); chk_cuda(shadow, "shadow");
  c10::cuda::CUDAGuard gd(p.device());
  TORCH_CHECK(shadow.scalar_type() == torch::kBFloat16 && shadow.numel() == p.numel(), "shadow");
  check(ts_cast_bf16(p.data_ptr<float>(), shadow.data_ptr(), p.numel(), stream()), "cast_bf16");
}

// ---- fused allreduce ----------------------------------------------------------------------------------------
// ptrs: CPU int64 [4, world] (in, param, shadow, flags); mc_*: multicast addresses or 0.
void fused_allreduce(const Tensor& ptrs, int64_t mc_in, int64_t mc_param, int64_t mc_shadow, std::optional<Tensor> m,
                     std::optional<Tensor> v, Tensor epochs, Tensor err, int64_t n, int64_t rank, int64_t world,
                     int64_t mode, bool two_shot, bool multicast, int64_t blocks, double lr, double b1, double b2,
                     double eps, double wd, double timeout_s, std::optional<Tensor> step_dev, int64_t wd_numel, bool bump_step, bool pdl) {
  TORCH_CHECK(!ptrs.is_cuda() && ptrs.scalar_type() == torch::kInt64 && ptrs.numel() == 4 * world, "ptrs: cpu int64 [4,world]");
  chk_cuda(epochs, "epochs"); chk_cuda(err, "err");
  c10::cuda::CUDAGuard gd(epochs.device());
  check(ts_fused_allreduce((const unsigned long long*)ptrs.data_ptr<int64_t>(), (unsigned long long)mc_in,
                           (unsigned long long)mc_param, (unsigned long long)mc_shadow,
                           m.has_value() ? m->data_ptr<float>() : nullptr, v.has_value() ? v->data_ptr<float>() : nullptr,
                           (unsigned int*)epochs.data_ptr<int>(), err.data_ptr<int>(), n, (int)rank, (int)world, (int)mode,
                           two_shot ? 1 : 0, multicast ? 1 : 0, (int)blocks, lr, b1, b2, eps, wd, timeout_s, stream(),
                           step_dev.has_value() ? step_dev->data_ptr<int>() : nullptr, (long long)wd_numel, bump_step ? 1 : 0, pdl ? 1 : 0),
        "fused_allreduce");
}

// ---- general wgmma GEMM (csrc/gemm2_wgmma.cu): C[M,N] (=|+=) op(A)·op(B) (+bias) ------------------------------------
// a_mn = false: A is [M,K] (K contiguous); true: A is [K,M] (M contiguous).  b_mn = false: B is [N,K]; true: B is [K,N].
// out: optional preallocated C (fp32 for accumulate = C += A·B, or any mode); out_fp32 selects the dtype of a fresh C.
Tensor gemm2(const Tensor& A, const Tensor& B, const std::optional<Tensor>& bias, std::optional<Tensor> out, bool a_mn, bool b_mn,
             bool out_fp32, bool accumulate, int64_t ctas, int64_t bn, int64_t max_ctas, const std::optional<Tensor>& gate,
             const std::vector<int64_t>& gate_cfg, const std::optional<Tensor>& done, const std::optional<Tensor>& gate_err,
             int64_t stream_handle, bool pdl, int64_t a_fold, int64_t b_fold, int64_t fold_cols) {
  // a_fold / b_fold: the operand is the 2-D storage view [fold, T * fold_cols] of a batch-major [fold, T, fold_cols] array that
  // is read as the time-major matrix [T * fold, fold_cols] (A: K-major, K = fold_cols;  B: MN-major, N = fold_cols)
  TORCH_CHECK(A.is_cuda() && B.is_cuda(), "gemm2: CUDA tensors");
  TORCH_CHECK(!(a_fold && b_fold) && (!a_fold || !a_mn) && (!b_fold || b_mn), "gemm2: one folded operand (K-major A or MN-major B)");
  TORCH_CHECK(A.scalar_type() == torch::kBFloat16 && B.scalar_type() == torch::kBFloat16, "gemm2: A/B must be bf16");
  TORCH_CHECK(A.dim() == 2 && B.dim() == 2 && A.stride(1) == 1 && B.stride(1) == 1, "gemm2: 2-D operands with unit inner stride");
  c10::cuda::CUDAGuard gd(A.device());
  if (a_fold) TORCH_CHECK(A.size(0) == a_fold && fold_cols > 0 && A.size(1) % fold_cols == 0, "gemm2: folded A must be [fold, T * fold_cols]");
  if (b_fold) TORCH_CHECK(B.size(0) == b_fold && fold_cols > 0 && B.size(1) % fold_cols == 0, "gemm2: folded B must be [fold, T * fold_cols]");
  const int M = a_fold ? (int)(a_fold * (A.size(1) / fold_cols)) : (a_mn ? A.size(1) : A.size(0));
  const int K = a_fold ? (int)fold_cols : (a_mn ? A.size(0) : A.size(1));
  const int N = b_fold ? (int)fold_cols : (b_mn ? B.size(1) : B.size(0));
  const int Kb = b_fold ? (int)(b_fold * (B.size(1) / fold_cols)) : (b_mn ? B.size(0) : B.size(1));
  TORCH_CHECK(K == Kb, "gemm2: contraction sizes differ (", K, " vs ", Kb, ")");
  Tensor C;
  if (out.has_value()) {
    C = *out;
    TORCH_CHECK(C.is_cuda() && C.dim() == 2 && C.size(0) == M && C.size(1) == N && C.stride(1) == 1, "gemm2: out must be [M,N]");
    TORCH_CHECK(C.scalar_type() == (out_fp32 || accumulate ? torch::kFloat32 : torch::kBFloat16), "gemm2: out dtype");
  } else {
    TORCH_CHECK(!accumulate, "gemm2: accumulate needs out=");
    C = torch::empty({M, N}, A.options().dtype(out_fp32 ? torch::kFloat32 : torch::kBFloat16));
  }
  const int out_mode = accumulate ? 2 : (C.scalar_type() == torch::kFloat32 ? 1 : 0);
  const unsigned int* gp = nullptr;
  int gcfg[7] = {0, 0, 0, 0, 1, 0, 0};
  if (gate.has_value()) {
    TORCH_CHECK(gate->is_cuda() && gate->scalar_type() == torch::kInt32 && gate_cfg.size() == 7, "gemm2: gate int32 cuda + 7 config ints");
    gp = (const unsigned int*)gate->data_ptr<int>();
    for (int i = 0; i < 7; ++i) gcfg[i] = (int)gate_cfg[i];
  }
  unsigned int* dp = nullptr;
  if (done.has_value()) { TORCH_CHECK(done->is_cuda() && done->scalar_type() == torch::kInt32, "gemm2: done int32 cuda"); dp = (unsigned int*)done->data_ptr<int>(); }
  check(ts_gemm2(A.data_ptr(), B.data_ptr(), C.data_ptr(), fptr(bias), M, N, K, (int)A.stride(0), (int)B.stride(0), (int)C.stride(0),
                 a_mn ? 1 : 0, b_mn ? 1 : 0, out_mode, (int)ctas, (int)bn, A.device().index(), (int)max_ctas, gp, gcfg, dp,
                 gate_err.has_value() ? gate_err->data_ptr<int>() : nullptr, pdl ? 1 : 0, (int)a_fold, (int)b_fold, (int)fold_cols,
                 stream_handle ? (cudaStream_t)stream_handle : stream()), "gemm2");
  return C;
}

// ---- any-shape CUDA-core GEMM (csrc/gemm_generic.cu): C = beta*C + A·B, A [M,K] / B [K,N] with arbitrary strides --------------
Tensor gemm_generic(const Tensor& A, const Tensor& B, const std::optional<Tensor>& bias, std::optional<Tensor> out, bool out_fp32, double beta) {
  TORCH_CHECK(A.is_cuda() && B.is_cuda() && A.dim() == 2 && B.dim() == 2 && A.size(1) == B.size(0), "gemm_generic: A [M,K] x B [K,N]");
  c10::cuda::CUDAGuard gd(A.device());
  const int M = A.size(0), K = A.size(1), N = B.size(1);
  Tensor C;
  if (out.has_value()) {
    C = *out;
    TORCH_CHECK(C.is_cuda() && C.dim() == 2 && C.size(0) == M && C.size(1) == N && C.stride(1) == 1, "gemm_generic: out [M,N]");
  } else {
    TORCH_CHECK(beta == 0.0, "gemm_generic: beta needs out=");
    C = torch::empty({M, N}, A.options().dtype(out_fp32 ? torch::kFloat32 : A.scalar_type()));
  }
  check(ts_gemm_generic(A.data_ptr(), B.data_ptr(), C.data_ptr(), fptr(bias), M, N, K, A.stride(0), A.stride(1), B.stride(0), B.stride(1),
                        C.stride(0), is_bf16(A), is_bf16(B), is_bf16(C), (float)beta, stream()), "gemm_generic");
  return C;
}

// ---- persistent wgmma LSTM sequence kernels ------------------------------------------------------------------
// gx [T,B,4H] bf16 (x·Wx^T, no bias), w_h [4H,H] bf16, bias fp32 [4H], h0 bf16 [B,H], c0 fp32 [B,H]
// -> h_seq [T+1,B,H] bf16 (row 0 = h0), c_seq [T+1,B,H] fp32, act [T,B,4H] bf16
// reverse: time runs from T-1 down to 0; h_seq / c_seq row t = the state after time t, row T = h0 / c0.
// in_gate (wavefront): completion counters of the GEMM that is still producing gx while this kernel runs (see SeqParams);
// extra_signal: one more arrival after the last step, for a gated GEMM that consumes h_seq.
std::vector<Tensor> lstm_seq_fwd(const Tensor& gx, const Tensor& w_h, const Tensor& bias, const Tensor& h0,
                                 const Tensor& c0, Tensor sync_ws, int64_t variant, std::optional<Tensor> dbg,
                                 std::optional<Tensor> in_gate, int64_t in_gate_tiles_n, bool extra_signal,
                                 const std::optional<Tensor>& lengths, bool reverse, const std::optional<Tensor>& drop_step,
                                 const std::vector<int64_t>& drop_desc) {
  chk_cuda(gx, "gx"); chk_cuda(w_h, "w_h"); chk_cuda(bias, "bias"); chk_cuda(h0, "h0"); chk_cuda(c0, "c0");
  c10::cuda::CUDAGuard gd(gx.device());
  int T = gx.size(0), B = gx.size(1), H = gx.size(2) / 4;
  const int* lp = lengths_ptr(lengths, B, gx);
  const int rev = direction_flag(reverse, in_gate, extra_signal);
  unsigned int dd[5];
  const int* ds = drop_args(drop_step, drop_desc, gx, dd);
  Tensor h_drop = ds ? torch::empty({T, B, H}, gx.options()) : Tensor();
  auto h_seq = torch::empty({T + 1, B, H}, gx.options());
  auto c_seq = torch::empty({T + 1, B, H}, c0.options());
  auto act = torch::empty({T, B, 4 * H}, gx.options());
  // streamed-operand images: [T+1][tiles_m][H/64][128][64] bf16, 128B-swizzled; slot 0 (= h0) and h_seq[0] / c_seq[0] /
  // the step counters are written by the launcher's prologue kernel
  const int tiles_m = (B + 127) / 128, nkb = H / 64;
  auto tiled = torch::empty({(int64_t)(T + 1), tiles_m, nkb, 128, 64}, gx.options());
  TORCH_CHECK(h0.scalar_type() == torch::kBFloat16 && c0.scalar_type() == torch::kFloat32, "h0 bf16 / c0 fp32");
  check(ts_lstm_seq_fwd(gx.data_ptr(), w_h.data_ptr(), bias.data_ptr<float>(), h_seq.data_ptr(), c_seq.data_ptr<float>(),
                        act.data_ptr(), c0.data_ptr<float>(), dbg.has_value() ? dbg->data_ptr() : nullptr, tiled.data_ptr(), T, B, H,
                        (unsigned int*)sync_ws.data_ptr<int>(), (int)variant, stream(), h0.data_ptr(),
                        in_gate.has_value() ? (const unsigned int*)in_gate->data_ptr<int>() : nullptr, (int)in_gate_tiles_n,
                        extra_signal ? 1 : 0, 0, lp, rev, ds ? h_drop.data_ptr() : nullptr, ds, dd), "lstm_seq_fwd");
  if (ds) return {h_seq, c_seq, act, h_drop};
  return {h_seq, c_seq, act};
}

// dh_seq [T,B,H] bf16 (grad wrt every h_t from above; None when only h_T is used downstream), w_hT [H,4H] bf16 (transposed recurrent weights),
// act/c_seq from forward, dhT fp32 [B,H] / dcT fp32 [B,H] extra grads into the final state (may be zeros)
// -> dpre [T,B,4H] bf16, dh0 fp32 [B,H], dc0 fp32 [B,H]
std::vector<Tensor> lstm_seq_bwd(const std::optional<Tensor>& dh_seq, const Tensor& w_hT, const Tensor& act, const Tensor& c_seq,
                                 const Tensor& dhT, const Tensor& dcT, Tensor sync_ws, int64_t variant,
                                 std::optional<Tensor> dbg, std::optional<Tensor> in_gate, int64_t in_gate_tiles_n, bool extra_signal,
                                 const std::optional<Tensor>& lengths, bool reverse, const std::optional<Tensor>& drop_step,
                                 const std::vector<int64_t>& drop_desc) {
  if (dh_seq.has_value()) chk_cuda(*dh_seq, "dh_seq");
  chk_cuda(w_hT, "w_hT"); chk_cuda(act, "act"); chk_cuda(c_seq, "c_seq");
  c10::cuda::CUDAGuard gd(act.device());
  int T = act.size(0), B = act.size(1), H = act.size(2) / 4;
  const int* lp = lengths_ptr(lengths, B, act);
  const int rev = direction_flag(reverse, in_gate, extra_signal);
  unsigned int dd[5];
  const int* ds = drop_args(drop_step, drop_desc, act, dd);
  auto dpre = torch::empty_like(act);
  auto dh0 = dhT.clone();
  auto dc0 = dcT.clone();
  const int tiles_m = (B + 127) / 128;
  auto tiled = torch::empty({(int64_t)T, tiles_m, 4 * H / 64, 128, 64}, act.options());   // dG images, written by the kernel
  check(ts_lstm_seq_bwd(dh_seq.has_value() ? dh_seq->data_ptr() : nullptr, w_hT.data_ptr(), act.data_ptr(), c_seq.data_ptr<float>(), dpre.data_ptr(),
                        dh0.data_ptr<float>(), dc0.data_ptr<float>(), dbg.has_value() ? dbg->data_ptr() : nullptr, tiled.data_ptr(), T, B, H,
                        (unsigned int*)sync_ws.data_ptr<int>(), (int)variant, stream(),
                        in_gate.has_value() ? (const unsigned int*)in_gate->data_ptr<int>() : nullptr, (int)in_gate_tiles_n,
                        extra_signal ? 1 : 0, 0, lp, rev, ds, dd), "lstm_seq_bwd");
  return {dpre, dh0, dc0};
}

// Wavefront variants: every buffer is preallocated by the caller (on the main stream, BEFORE it forks side streams) and the
// launch goes to an explicit stream - the caching allocator never sees a side stream.
void lstm_seq_fwd_into(const Tensor& gx, const Tensor& w_h, const Tensor& bias, const Tensor& h0, const Tensor& c0, Tensor h_seq,
                       Tensor c_seq, Tensor act, Tensor tiled, Tensor sync_ws, int64_t variant, std::optional<Tensor> in_gate,
                       int64_t in_gate_tiles_n, bool extra_signal, int64_t stream_handle, int64_t launch_flags,
                       const std::optional<Tensor>& lengths, bool reverse, const std::optional<Tensor>& h_drop,
                       const std::optional<Tensor>& drop_step, const std::vector<int64_t>& drop_desc) {
  chk_cuda(gx, "gx"); chk_cuda(w_h, "w_h"); chk_cuda(bias, "bias"); chk_cuda(h0, "h0"); chk_cuda(c0, "c0");
  chk_cuda(h_seq, "h_seq"); chk_cuda(c_seq, "c_seq"); chk_cuda(act, "act"); chk_cuda(tiled, "tiled");
  c10::cuda::CUDAGuard gd(gx.device());
  int T = gx.size(0), B = gx.size(1), H = gx.size(2) / 4;
  const int* lp = lengths_ptr(lengths, B, gx);
  const int rev = direction_flag(reverse, in_gate, extra_signal);
  TORCH_CHECK(h_seq.numel() == (int64_t)(T + 1) * B * H && c_seq.numel() == h_seq.numel() && act.numel() == gx.numel(), "lstm_seq_fwd_into: buffer sizes");
  TORCH_CHECK(tiled.numel() == (int64_t)(T + 1) * ((B + 127) / 128) * 128 * H, "lstm_seq_fwd_into: tile-image buffer size");
  TORCH_CHECK(h0.scalar_type() == torch::kBFloat16 && c0.scalar_type() == torch::kFloat32, "h0 bf16 / c0 fp32");
  unsigned int dd[5];
  const int* ds = drop_args(drop_step, drop_desc, gx, dd);
  if (ds) {
    TORCH_CHECK(h_drop.has_value(), "lstm_seq_fwd_into: dropout needs h_drop");
    chk_cuda(*h_drop, "h_drop");
    TORCH_CHECK(h_drop->scalar_type() == gx.scalar_type() && h_drop->numel() == (int64_t)T * B * H, "lstm_seq_fwd_into: h_drop [T,B,H]");
  }
  check(ts_lstm_seq_fwd(gx.data_ptr(), w_h.data_ptr(), bias.data_ptr<float>(), h_seq.data_ptr(), c_seq.data_ptr<float>(),
                        act.data_ptr(), c0.data_ptr<float>(), nullptr, tiled.data_ptr(), T, B, H, (unsigned int*)sync_ws.data_ptr<int>(),
                        (int)variant, stream_handle ? (cudaStream_t)stream_handle : stream(), h0.data_ptr(),
                        in_gate.has_value() ? (const unsigned int*)in_gate->data_ptr<int>() : nullptr, (int)in_gate_tiles_n,
                        extra_signal ? 1 : 0, (int)launch_flags, lp, rev, ds ? h_drop->data_ptr() : nullptr, ds, dd), "lstm_seq_fwd_into");
}

// h_seq[0] <- h0, c_seq[0] <- c0 (reverse: row T), tile image of h0, step counters <- 0 (what lstm_seq_fwd does first unless
// launch_flags bit 0)
void lstm_seq_prologue(const Tensor& h0, const Tensor& c0, Tensor h_seq, Tensor c_seq, Tensor tiled, Tensor sync_ws, bool reverse) {
  chk_cuda(h0, "h0"); chk_cuda(c0, "c0"); chk_cuda(h_seq, "h_seq"); chk_cuda(c_seq, "c_seq"); chk_cuda(tiled, "tiled");
  c10::cuda::CUDAGuard gd(h0.device());
  TORCH_CHECK(h0.scalar_type() == torch::kBFloat16 && c0.scalar_type() == torch::kFloat32 && h0.dim() == 2, "h0 bf16 [B,H] / c0 fp32");
  TORCH_CHECK(h_seq.scalar_type() == torch::kBFloat16 && h_seq.numel() % h0.numel() == 0 && h_seq.numel() >= h0.numel() &&
              c_seq.numel() == h_seq.numel(), "lstm_seq_prologue: h_seq bf16 / c_seq [T+1,B,H]");
  const int64_t init_off = reverse ? h_seq.numel() - h0.numel() : 0;       // row T
  check(ts_lstm_seq_prologue(h0.data_ptr(), c0.data_ptr<float>(), (at::BFloat16*)h_seq.data_ptr() + init_off, c_seq.data_ptr<float>() + init_off, tiled.data_ptr(),
                             (unsigned int*)sync_ws.data_ptr<int>(), (int)h0.size(0), (int)h0.size(1), stream()), "lstm_seq_prologue");
}

void lstm_seq_bwd_into(const std::optional<Tensor>& dh_seq, const Tensor& w_hT, const Tensor& act, const Tensor& c_seq, Tensor dpre,
                       Tensor dh0, Tensor dc0, Tensor tiled, Tensor sync_ws, int64_t variant, std::optional<Tensor> in_gate,
                       int64_t in_gate_tiles_n, bool extra_signal, int64_t stream_handle, int64_t launch_flags,
                       const std::optional<Tensor>& lengths, bool reverse, const std::optional<Tensor>& drop_step,
                       const std::vector<int64_t>& drop_desc) {
  chk_cuda(w_hT, "w_hT"); chk_cuda(act, "act"); chk_cuda(c_seq, "c_seq"); chk_cuda(dpre, "dpre"); chk_cuda(dh0, "dh0"); chk_cuda(dc0, "dc0");
  c10::cuda::CUDAGuard gd(act.device());
  int T = act.size(0), B = act.size(1), H = act.size(2) / 4;
  const int* lp = lengths_ptr(lengths, B, act);
  const int rev = direction_flag(reverse, in_gate, extra_signal);
  TORCH_CHECK(dpre.numel() == act.numel() && tiled.numel() == (int64_t)T * ((B + 127) / 128) * 128 * 4 * H, "lstm_seq_bwd_into: buffer sizes");
  TORCH_CHECK(dh0.scalar_type() == torch::kFloat32 && dc0.scalar_type() == torch::kFloat32 && dh0.numel() == (int64_t)B * H && dc0.numel() == (int64_t)B * H, "dh0/dc0 fp32 [B,H]");
  unsigned int dd[5];
  const int* ds = drop_args(drop_step, drop_desc, act, dd);
  check(ts_lstm_seq_bwd(dh_seq.has_value() ? dh_seq->data_ptr() : nullptr, w_hT.data_ptr(), act.data_ptr(), c_seq.data_ptr<float>(), dpre.data_ptr(),
                        dh0.data_ptr<float>(), dc0.data_ptr<float>(), nullptr, tiled.data_ptr(), T, B, H, (unsigned int*)sync_ws.data_ptr<int>(),
                        (int)variant, stream_handle ? (cudaStream_t)stream_handle : stream(),
                        in_gate.has_value() ? (const unsigned int*)in_gate->data_ptr<int>() : nullptr, (int)in_gate_tiles_n,
                        extra_signal ? 1 : 0, (int)launch_flags, lp, rev, ds, dd), "lstm_seq_bwd_into");
}

}  // namespace

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.doc() = "lstm_tensorspark_b200 sm_90a kernels";
  m.def("lstm_pointwise_fwd", &lstm_pointwise_fwd, py::arg("pre"), py::arg("bias"), py::arg("c_prev"), py::arg("h_prev") = py::none(),
        py::arg("lengths") = py::none(), py::arg("t") = 0);
  m.def("transpose01", &transpose01);
  m.def("transpose2d", &transpose2d);
  m.def("colsum_bf16", &colsum_bf16);
  m.def("colsum_bf16_into", &colsum_bf16_into, py::arg("x"), py::arg("out"), py::arg("overwrite"), py::arg("pdl") = false,
        py::arg("col0") = 0, py::arg("ncols") = 0, py::arg("max_ctas") = 0);
  m.def("lstm_seq_cluster_probe", [](int64_t c) { return ts_lstm_seq_cluster_probe((int)c); });
  // (ring stages, batch tiles per CTA, streamed weights, forward K-split) of the persistent kernel for these arguments
  m.def("lstm_seq_config", [](bool bwd, int64_t H, int64_t B, int64_t variant) {
    int out[4];
    check(ts_lstm_seq_config(bwd ? 1 : 0, (int)H, (int)B, (int)variant, out), "lstm_seq_config");
    return std::make_tuple(out[0], out[1], out[2] != 0, out[3] != 0);
  }, py::arg("bwd"), py::arg("H"), py::arg("B"), py::arg("variant") = 0);
  m.def("lstm_pointwise_bwd", &lstm_pointwise_bwd, py::arg("dh_a"), py::arg("dh_b"), py::arg("dc_in"), py::arg("act"), py::arg("c_prev"),
        py::arg("c_new"), py::arg("lengths") = py::none(), py::arg("t") = 0);
  m.def("xent_rows", &xent_rows);
  m.def("head_fwd", &head_fwd);
  m.def("head_bwd", &head_bwd, py::arg("h"), py::arg("W"), py::arg("dlogits"), py::arg("dloss"), py::arg("dW"), py::arg("db"),
        py::arg("accumulate") = false);
  m.def("flat_adam", &flat_adam, py::arg("p"), py::arg("g"), py::arg("m"), py::arg("v"), py::arg("shadow"), py::arg("lr_t"),
        py::arg("b1"), py::arg("b2"), py::arg("eps"), py::arg("wd"), py::arg("gscale"), py::arg("step_dev") = py::none(),
        py::arg("wd_numel") = -1);
  m.def("flat_sgd", &flat_sgd, py::arg("p"), py::arg("g"), py::arg("shadow"), py::arg("lr"), py::arg("wd"), py::arg("gscale"),
        py::arg("wd_numel") = -1);
  m.def("cast_bf16", &cast_bf16);
  m.def("fused_allreduce", &fused_allreduce, py::arg("ptrs"), py::arg("mc_in"), py::arg("mc_param"), py::arg("mc_shadow"), py::arg("m"),
        py::arg("v"), py::arg("epochs"), py::arg("err"), py::arg("n"), py::arg("rank"), py::arg("world"), py::arg("mode"),
        py::arg("two_shot"), py::arg("multicast"), py::arg("blocks"), py::arg("lr"), py::arg("b1"), py::arg("b2"), py::arg("eps"),
        py::arg("wd"), py::arg("timeout_s"), py::arg("step_dev") = py::none(), py::arg("wd_numel") = -1, py::arg("bump_step") = true,
        py::arg("pdl") = false);
  m.def("ar_bump_step", [](Tensor step_dev) {
    TORCH_CHECK(step_dev.is_cuda() && step_dev.scalar_type() == torch::kInt32, "ar_bump_step: int32 cuda tensor");
    c10::cuda::CUDAGuard gd(step_dev.device());
    check(ts_ar_bump_step(step_dev.data_ptr<int>(), stream()), "ar_bump_step");
  });
  m.def("ar_max_blocks", []() { return ts_ar_max_blocks(); });
  m.def("ar_flag_words", []() { return ts_ar_flag_words(); });
  m.def("ar_slots", []() { return ts_ar_slots(); });
  m.def("gemm_generic", &gemm_generic, py::arg("A"), py::arg("B"), py::arg("bias") = py::none(), py::arg("out") = py::none(),
        py::arg("out_fp32") = false, py::arg("beta") = 0.0);
  m.def("gemm2", &gemm2, py::arg("A"), py::arg("B"), py::arg("bias") = py::none(), py::arg("out") = py::none(), py::arg("a_mn") = false,
        py::arg("b_mn") = false, py::arg("out_fp32") = false, py::arg("accumulate") = false, py::arg("ctas") = 2, py::arg("bn") = 256,
        py::arg("max_ctas") = 0, py::arg("gate") = py::none(), py::arg("gate_cfg") = std::vector<int64_t>{}, py::arg("done") = py::none(),
        py::arg("gate_err") = py::none(), py::arg("stream") = 0, py::arg("pdl") = false, py::arg("a_fold") = 0, py::arg("b_fold") = 0,
        py::arg("fold_cols") = 0);
  m.def("lstm_seq_fwd", &lstm_seq_fwd, py::arg("gx"), py::arg("w_h"), py::arg("bias"), py::arg("h0"), py::arg("c0"),
        py::arg("sync_ws"), py::arg("variant") = 0, py::arg("dbg") = py::none(), py::arg("in_gate") = py::none(),
        py::arg("in_gate_tiles_n") = 0, py::arg("extra_signal") = false, py::arg("lengths") = py::none(), py::arg("reverse") = false,
        py::arg("drop_step") = py::none(), py::arg("drop_desc") = std::vector<int64_t>{});
  m.def("lstm_seq_fwd_into", &lstm_seq_fwd_into, py::arg("gx"), py::arg("w_h"), py::arg("bias"), py::arg("h0"), py::arg("c0"),
        py::arg("h_seq"), py::arg("c_seq"), py::arg("act"), py::arg("tiled"), py::arg("sync_ws"), py::arg("variant"),
        py::arg("in_gate") = py::none(), py::arg("in_gate_tiles_n") = 0, py::arg("extra_signal") = false, py::arg("stream") = 0,
        py::arg("launch_flags") = 0, py::arg("lengths") = py::none(), py::arg("reverse") = false, py::arg("h_drop") = py::none(),
        py::arg("drop_step") = py::none(), py::arg("drop_desc") = std::vector<int64_t>{});
  m.def("lstm_seq_prologue", &lstm_seq_prologue, py::arg("h0"), py::arg("c0"), py::arg("h_seq"), py::arg("c_seq"), py::arg("tiled"),
        py::arg("sync_ws"), py::arg("reverse") = false);
  m.def("lstm_seq_bwd_into", &lstm_seq_bwd_into, py::arg("dh_seq"), py::arg("w_hT"), py::arg("act"), py::arg("c_seq"), py::arg("dpre"),
        py::arg("dh0"), py::arg("dc0"), py::arg("tiled"), py::arg("sync_ws"), py::arg("variant"), py::arg("in_gate") = py::none(),
        py::arg("in_gate_tiles_n") = 0, py::arg("extra_signal") = false, py::arg("stream") = 0, py::arg("launch_flags") = 0,
        py::arg("lengths") = py::none(), py::arg("reverse") = false, py::arg("drop_step") = py::none(),
        py::arg("drop_desc") = std::vector<int64_t>{});
  m.def("lstm_seq_bwd", &lstm_seq_bwd, py::arg("dh_seq"), py::arg("w_hT"), py::arg("act"), py::arg("c_seq"), py::arg("dhT"),
        py::arg("dcT"), py::arg("sync_ws"), py::arg("variant") = 0, py::arg("dbg") = py::none(), py::arg("in_gate") = py::none(),
        py::arg("in_gate_tiles_n") = 0, py::arg("extra_signal") = false, py::arg("lengths") = py::none(), py::arg("reverse") = false,
        py::arg("drop_step") = py::none(), py::arg("drop_desc") = std::vector<int64_t>{});
  m.def("dropout", &dropout, py::arg("x"), py::arg("step"), py::arg("desc"), py::arg("t0") = 0);
}
