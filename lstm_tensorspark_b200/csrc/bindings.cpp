// Python bindings for the sm_90a kernels (the only translation unit that sees torch headers).
// Every function validates device / dtype / contiguity, takes the CURRENT torch CUDA stream (so the kernels
// are stream-ordered with the rest of the step and capturable in CUDA graphs) and forwards raw pointers to the
// C-ABI launchers defined next to the kernels.
#include <torch/extension.h>
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAException.h>
#include <cuda_runtime.h>

#include <cmath>
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
                 cudaStream_t, int*, long long, const float*);
int ts_flat_sgd(float*, const float*, void*, long long, float, float, float, cudaStream_t, long long, const float*);
long long ts_flat_grad_norm_scratch(long long);
int ts_flat_grad_norm(const float*, const float*, long long, float, float, long long, float, double*, float*, cudaStream_t);
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
int ts_head_bwd(const void*, const float*, const float*, const float*, void*, float*, float*, int, int, int, int, int, int, cudaStream_t);
int ts_head_step_fwd_generic_parts(int);
int ts_head_step_fwd(const void*, int, int, const float*, const float*, const long long*, const int*, float*, float*, float*, int*,
                     unsigned int*, float*, int*, int*, int, int, int, int, int*, cudaStream_t);
long long ts_head_step_bwd_scratch(int, int, int);
int ts_head_step_bwd_tickets(int);
int ts_head_step_bwd(const void*, const float*, const float*, const float*, void*, float*, float*, float*, unsigned int*, int, int, int,
                     int, int, int, cudaStream_t);
int ts_vocab_head_parts(int);
int ts_vocab_head_blocks(int);
int ts_vocab_head_fwd(const void*, const void*, int, const float*, const long long*, const int*, void*, float*, float*, int*, unsigned int*,
                      float*, int*, int*, int, int, int, int, int, cudaStream_t);
int ts_vocab_head_dlogits(const void*, const void*, int, const float*, const long long*, const int*, const float*, const float*, const int*,
                          void*, int, int, int, int, int, int, int, cudaStream_t);
int ts_vocab_head_colsum(const void*, float*, int, int, int, cudaStream_t);
int ts_vocab_sample(const void*, const void*, int, const float*, float, unsigned int, int*, const int*, void*, int*, unsigned int*, int*,
                    float*, int*, float*, int, int, int, int, int, int, cudaStream_t);
int ts_vocab_sample_logits(const float*, const float*, float, unsigned int, int*, const int*, void*, int*, unsigned int*, int*, float*, int*,
                           float*, int, int, int, int, cudaStream_t);
int ts_vocab_head_logits(const void*, const void*, int, const float*, float*, int, int, int, int, cudaStream_t);
int ts_vocab_threshold(const float*, int, int, int, double, float, float*, cudaStream_t);
int ts_gemm_generic(const void*, const void*, void*, const float*, int, int, int, long long, long long, long long, long long, long long,
                    int, int, int, float, cudaStream_t);
int ts_gemm2(const void*, const void*, void*, const float*, int, int, int, int, int, int, int, int, int, int, int, int, int,
             const unsigned int*, const int*, unsigned int*, int*, int, int, int, int, float*, int, cudaStream_t);
int ts_lstm_seq_fwd(const void*, const void*, const float*, const void*, const float*, void*, const float*, void*, void*, int,
                    int, int, unsigned int*, int, cudaStream_t, const void*, const unsigned int*, int, int, int, const int*, int,
                    void*, const int*, const unsigned int*);
int ts_lstm_seq_bwd(const void*, const void*, const void*, const float*, const void*, float*, float*, void*, void*, int,
                    int, int, unsigned int*, int, cudaStream_t, const unsigned int*, int, int, int, const int*, int,
                    const int*, const unsigned int*);
int ts_dropout(const void*, void*, int, int, int, int, int, const int*, const unsigned int*, cudaStream_t);
int ts_weight_drop_grad(const float*, float*, int, int, int, const int*, const unsigned int*, cudaStream_t);
int ts_lstm_seq_prologue(const void*, const float*, void*, float*, void*, unsigned int*, int, int, cudaStream_t);
int ts_seq_pool_fwd(const void*, int, const int*, const float*, int, int, int, int, float*, int*, cudaStream_t);
int ts_seq_pool_attn_scores(float*, const float*, const float*, const int*, int, int, int, float*, int, cudaStream_t);
int ts_seq_pool_attn_bwd(const void*, int, const float*, const float*, const float*, const float*, const int*, int, int, int, int,
                         float*, void*, float*, unsigned int*, float*, float*, int, int, cudaStream_t);
int ts_seq_pool_bwd(const float*, const int*, const int*, const float*, const float*, int, int, int, int, void*, int, cudaStream_t);
void ts_embed_scratch_numel(long long, long long, long long, long long*);
int ts_embed_fwd(const void*, int, const int*, const int*, int, int, int, int, void*, const int*, const unsigned int*, const int*,
                 const unsigned int*, cudaStream_t);
int ts_embed_bwd(const void*, int, const int*, const int*, int, int, int, int, float*, int, int*, int*, float*, const int*,
                 const unsigned int*, const int*, const unsigned int*, cudaStream_t);
int ts_embed_bwd_launches();
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

// Weight drop's gradient: dst (+)= src * mask * scale over fp32 [R, H] (R = 4H rows of W_h), the mask of `desc` at time 0, as
// `dropout` draws it for the [1, R, H] weight image.  src may be dst when accumulate is false (in place).
void weight_drop_grad(const Tensor& src, Tensor dst, const Tensor& step, const std::vector<int64_t>& desc, bool accumulate) {
  chk_cuda(src, "src"); chk_cuda(dst, "dst");
  TORCH_CHECK(src.scalar_type() == torch::kFloat32 && dst.scalar_type() == torch::kFloat32 && src.dim() == 2 && src.sizes() == dst.sizes(),
              "weight_drop_grad: src and dst must be fp32 [R, H] of the same shape");
  TORCH_CHECK(!accumulate || src.data_ptr() != dst.data_ptr(), "weight_drop_grad: in place only in overwrite mode");
  c10::cuda::CUDAGuard g(src.device());
  unsigned int dd[5];
  const int* ds = drop_args(step, desc, src, dd);
  TORCH_CHECK(dd[4] == 0, "weight_drop_grad: the weight mask has no row offset (row0 = 0)");
  check(ts_weight_drop_grad(src.data_ptr<float>(), dst.data_ptr<float>(), (int)src.size(0), (int)src.size(1), accumulate ? 1 : 0, ds, dd,
                            stream()), "weight_drop_grad");
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
// acc_w / acc_b: add into dW / db instead of overwriting them.
Tensor head_bwd(const Tensor& h, const Tensor& W, const Tensor& dlogits, const std::optional<Tensor>& dloss, Tensor dW, Tensor db,
                bool acc_w, bool acc_b) {
  chk_cuda(h, "h"); chk_cuda(W, "W"); chk_cuda(dlogits, "dlogits"); chk_cuda(dW, "dW"); chk_cuda(db, "db");
  c10::cuda::CUDAGuard g(h.device());
  const int B = h.size(0), H = h.size(1), C = W.size(1);
  TORCH_CHECK(dW.scalar_type() == torch::kFloat32 && db.scalar_type() == torch::kFloat32 && dW.numel() == (int64_t)H * C && db.numel() == C, "head_bwd: dW/db");
  TORCH_CHECK(dlogits.scalar_type() == torch::kFloat32 && dlogits.numel() == (int64_t)B * C, "head_bwd: dlogits fp32 [B,C]");
  auto dh = torch::empty_like(h);
  check(ts_head_bwd(h.data_ptr(), W.data_ptr<float>(), dlogits.data_ptr<float>(), fptr(dloss), dh.data_ptr(), dW.data_ptr<float>(),
                    db.data_ptr<float>(), B, H, C, is_bf16(h), acc_w ? 1 : 0, acc_b ? 1 : 0, stream()), "head_bwd");
  return dh;
}

// Per-step head (csrc/head_wgmma.cu): h [T·B, H] = the rows of h_seq [T,B,H] (row pitch = stride(0)), labels int64 [B,T], optional
// lengths int32 [B] -> logits [B,T,C], dlogits [T·B,C] (row order of h), loss (mean over counted rows), correct, N, and whether the
// tensor-core kernel ran.  Nothing is read back to the host.
std::vector<Tensor> head_step_fwd(const Tensor& h, const Tensor& W, const Tensor& bias, const Tensor& labels,
                                  const std::optional<Tensor>& lengths, int64_t T) {
  TORCH_CHECK(h.is_cuda() && h.dim() == 2 && h.stride(1) == 1, "head_step_fwd: h [T*B,H] with unit inner stride");
  chk_cuda(W, "W"); chk_cuda(bias, "bias"); chk_cuda(labels, "labels");
  c10::cuda::CUDAGuard g(h.device());
  const int R = h.size(0), H = h.size(1), C = W.size(1);
  TORCH_CHECK(T >= 1 && R % T == 0, "head_step_fwd: rows must be T*B");
  const int B = R / (int)T;
  TORCH_CHECK(W.size(0) == H && W.scalar_type() == torch::kFloat32 && bias.scalar_type() == torch::kFloat32 && bias.numel() == C, "head W/b");
  TORCH_CHECK(labels.scalar_type() == torch::kInt64 && labels.dim() == 2 && labels.size(0) == B && labels.size(1) == T, "labels int64 [B,T]");
  const int* lp = nullptr;
  if (lengths.has_value()) {
    chk_cuda(*lengths, "lengths");
    TORCH_CHECK(lengths->scalar_type() == torch::kInt32 && lengths->numel() == B, "lengths int32 [B]");
    lp = lengths->data_ptr<int>();
  }
  auto fo = torch::TensorOptions().device(h.device()).dtype(torch::kFloat32);
  auto io = fo.dtype(torch::kInt32);
  auto logits = torch::empty({B, (int64_t)T, C}, fo), dlogits = torch::empty({R, C}, fo);
  const int parts = ts_head_step_fwd_generic_parts(R);         // the larger of the two paths' grids
  auto part_loss = torch::empty({parts}, fo);
  auto ints = torch::zeros({parts + 4}, io);                   // [parts] per-CTA counts, ticket, correct, N
  auto loss = torch::empty({1}, fo);
  Tensor hc = h;
  if (h.scalar_type() != torch::kBFloat16 && h.stride(0) != H) hc = h.contiguous();
  int used_tc = 0;
  int rc = ts_head_step_fwd(hc.data_ptr(), (int)hc.stride(0), is_bf16(hc), W.data_ptr<float>(), bias.data_ptr<float>(),
                            (const long long*)labels.data_ptr<int64_t>(), lp, logits.data_ptr<float>(), dlogits.data_ptr<float>(),
                            part_loss.data_ptr<float>(), ints.data_ptr<int>(), (unsigned int*)(ints.data_ptr<int>() + parts),
                            loss.data_ptr<float>(), ints.data_ptr<int>() + parts + 1, ints.data_ptr<int>() + parts + 2, (int)T, B, H, C,
                            &used_tc, stream());
  if (rc == -2) {                                              // a strided bf16 h the tensor-core kernel did not take
    hc = h.contiguous();
    rc = ts_head_step_fwd(hc.data_ptr(), H, 1, W.data_ptr<float>(), bias.data_ptr<float>(), (const long long*)labels.data_ptr<int64_t>(),
                          lp, logits.data_ptr<float>(), dlogits.data_ptr<float>(), part_loss.data_ptr<float>(), ints.data_ptr<int>(),
                          (unsigned int*)(ints.data_ptr<int>() + parts), loss.data_ptr<float>(), ints.data_ptr<int>() + parts + 1,
                          ints.data_ptr<int>() + parts + 2, (int)T, B, H, C, &used_tc, stream());
  }
  check(rc, "head_step_fwd");
  return {logits, dlogits, loss, ints.narrow(0, parts + 1, 1), ints.narrow(0, parts + 2, 1),
          torch::full({1}, used_tc, torch::TensorOptions().dtype(torch::kInt32))};
}

// dh = (dloss * dlogits) W^T [T·B,H] (dtype of h), dW (+)= h^T (dloss * dlogits), db (+)= column sums: one launch, reduced in a
// fixed order (bitwise reproducible).  acc_w / acc_b: add into dW / db instead of overwriting them.
Tensor head_step_bwd(const Tensor& h, const Tensor& W, const Tensor& dlogits, const std::optional<Tensor>& dloss, Tensor dW, Tensor db,
                     bool acc_w, bool acc_b) {
  chk_cuda(h, "h"); chk_cuda(W, "W"); chk_cuda(dlogits, "dlogits"); chk_cuda(dW, "dW"); chk_cuda(db, "db");
  c10::cuda::CUDAGuard g(h.device());
  const int R = h.size(0), H = h.size(1), C = W.size(1);
  TORCH_CHECK(dW.scalar_type() == torch::kFloat32 && db.scalar_type() == torch::kFloat32 && dW.numel() == (int64_t)H * C && db.numel() == C, "head_step_bwd: dW/db");
  TORCH_CHECK(dlogits.scalar_type() == torch::kFloat32 && dlogits.numel() == (int64_t)R * C, "head_step_bwd: dlogits fp32 [R,C]");
  auto dh = torch::empty_like(h);
  auto fo = torch::TensorOptions().device(h.device()).dtype(torch::kFloat32);
  auto scratch = torch::empty({std::max<long long>(1, ts_head_step_bwd_scratch(R, H, C))}, fo);
  auto tickets = torch::zeros({ts_head_step_bwd_tickets(H)}, fo.dtype(torch::kInt32));
  check(ts_head_step_bwd(h.data_ptr(), W.data_ptr<float>(), dlogits.data_ptr<float>(), fptr(dloss), dh.data_ptr(), dW.data_ptr<float>(),
                         db.data_ptr<float>(), scratch.data_ptr<float>(), (unsigned int*)tickets.data_ptr<int>(), R, H, C, is_bf16(h),
                         acc_w ? 1 : 0, acc_b ? 1 : 0, stream()), "head_step_bwd");
  return dh;
}

// ---- large-vocabulary per-step head (csrc/head_vocab.cu) ------------------------------------------------------------
// h bf16 [T·B, H] packed time-major rows, Wb bf16 [H, C] (w_kmajor: the tied embedding table [C, H], read in place as a K-major
// operand; the flag is explicit because H == C would make the shapes ambiguous), bias fp32 [C], labels int64 [B,T], optional
// lengths int32 [B] (0 allowed), part: fp32 scratch of at least T·B * vocab_head_parts(C) * 4 elements -> lse [T·B], loss,
// correct, N.  No logits are stored and nothing is read back to the host.
int64_t vocab_classes(const Tensor& h, const Tensor& Wb, bool w_kmajor, const char* what) {
  TORCH_CHECK(h.dim() == 2 && Wb.dim() == 2 && h.scalar_type() == torch::kBFloat16 && Wb.scalar_type() == torch::kBFloat16 &&
              Wb.size(w_kmajor ? 1 : 0) == h.size(1), what, ": h bf16 [rows,H], Wb bf16 ", w_kmajor ? "[C,H]" : "[H,C]");
  TORCH_CHECK(!w_kmajor || (Wb.is_contiguous() && (uintptr_t)Wb.data_ptr() % 16 == 0), what, ": the table [C,H] must be packed and "
              "16-byte aligned (TMA)");
  return Wb.size(w_kmajor ? 0 : 1);
}

void vocab_head_check(const Tensor& h, const Tensor& Wb, bool w_kmajor, const Tensor& bias, const Tensor& labels, int64_t T) {
  chk_cuda(h, "h"); chk_cuda(Wb, "Wb"); chk_cuda(bias, "bias"); chk_cuda(labels, "labels");
  const int64_t R = h.size(0), H = h.size(1), C = vocab_classes(h, Wb, w_kmajor, "vocab head");
  TORCH_CHECK(H % 64 == 0 && C % 8 == 0 && C >= 8, "vocab head: H % 64 == 0 and C % 8 == 0");
  TORCH_CHECK(T >= 1 && R % T == 0 && R * std::max(C, H) < (int64_t(1) << 40) && R < (int64_t(1) << 31), "vocab head: rows must be T*B");
  TORCH_CHECK(bias.scalar_type() == torch::kFloat32 && bias.numel() == C && ((uintptr_t)bias.data_ptr() % 8) == 0, "vocab head: bias fp32 [C]");
  TORCH_CHECK(labels.scalar_type() == torch::kInt64 && labels.dim() == 2 && labels.size(0) == R / T && labels.size(1) == T, "labels int64 [B,T]");
}

std::vector<Tensor> vocab_head_fwd(const Tensor& h, const Tensor& Wb, bool w_kmajor, const Tensor& bias, const Tensor& labels,
                                   const std::optional<Tensor>& lengths, int64_t T, Tensor part) {
  vocab_head_check(h, Wb, w_kmajor, bias, labels, T);
  c10::cuda::CUDAGuard g(h.device());
  const int R = h.size(0), H = h.size(1), C = Wb.size(w_kmajor ? 0 : 1), B = R / (int)T;
  chk_cuda(part, "part");
  TORCH_CHECK(part.scalar_type() == torch::kFloat32 && part.numel() >= (int64_t)R * ts_vocab_head_parts(C) * 4 &&
              ((uintptr_t)part.data_ptr() % 16) == 0, "vocab head: part scratch");
  auto fo = torch::TensorOptions().device(h.device()).dtype(torch::kFloat32);
  const int blocks = ts_vocab_head_blocks(R);
  auto lse = torch::empty({R}, fo), part_loss = torch::empty({blocks}, fo), loss = torch::empty({1}, fo);
  auto ints = torch::zeros({blocks + 4}, fo.dtype(torch::kInt32));          // [blocks] per-block counts, ticket, correct, N
  int* ip = ints.data_ptr<int>();
  check(ts_vocab_head_fwd(h.data_ptr(), Wb.data_ptr(), w_kmajor ? 1 : 0, bias.data_ptr<float>(), (const long long*)labels.data_ptr<int64_t>(),
                          lengths_ptr(lengths, B, h), part.data_ptr(), lse.data_ptr<float>(), part_loss.data_ptr<float>(), ip,
                          (unsigned int*)(ip + blocks), loss.data_ptr<float>(), ip + blocks + 1, ip + blocks + 2, (int)T, B, H, C,
                          h.get_device(), stream()), "vocab_head_fwd");
  return {lse, loss, ints.narrow(0, blocks + 1, 1), ints.narrow(0, blocks + 2, 1)};
}

// dl [rows, C] bf16 <- (softmax - onehot) * dloss / N of rows [row0, row0 + rows) of h (0 at uncounted rows); lse, count: the forward's.
void vocab_head_dlogits(const Tensor& h, const Tensor& Wb, bool w_kmajor, const Tensor& bias, const Tensor& labels,
                        const std::optional<Tensor>& lengths, int64_t T, const Tensor& lse, const Tensor& count, const Tensor& dloss,
                        int64_t row0, int64_t rows, Tensor dl) {
  vocab_head_check(h, Wb, w_kmajor, bias, labels, T);
  c10::cuda::CUDAGuard g(h.device());
  const int R = h.size(0), H = h.size(1), C = Wb.size(w_kmajor ? 0 : 1), B = R / (int)T;
  chk_cuda(lse, "lse"); chk_cuda(count, "count"); chk_cuda(dloss, "dloss"); chk_cuda(dl, "dl");
  TORCH_CHECK(lse.scalar_type() == torch::kFloat32 && lse.numel() == R && count.scalar_type() == torch::kInt32 && count.numel() == 1 &&
              dloss.scalar_type() == torch::kFloat32 && dloss.numel() == 1, "vocab head: lse fp32 [R], count int32 [1], dloss fp32 [1]");
  TORCH_CHECK(rows >= 1 && row0 >= 0 && row0 + rows <= R && dl.scalar_type() == torch::kBFloat16 && dl.numel() >= rows * C,
              "vocab head: dl bf16 [rows, C]");
  check(ts_vocab_head_dlogits(h.data_ptr(), Wb.data_ptr(), w_kmajor ? 1 : 0, bias.data_ptr<float>(), (const long long*)labels.data_ptr<int64_t>(),
                              lengths_ptr(lengths, B, h), lse.data_ptr<float>(), dloss.data_ptr<float>(), count.data_ptr<int>(),
                              dl.data_ptr(), (int)T, B, H, C, (int)row0, (int)rows, h.get_device(), stream()), "vocab_head_dlogits");
}

// db [C] (+)= column sums of dl [rows, C] (bf16), summed in a fixed order.
void vocab_head_colsum(const Tensor& dl, Tensor db, bool accumulate) {
  chk_cuda(dl, "dl"); chk_cuda(db, "db");
  c10::cuda::CUDAGuard g(dl.device());
  TORCH_CHECK(dl.dim() == 2 && dl.scalar_type() == torch::kBFloat16 && dl.size(1) % 2 == 0 && db.scalar_type() == torch::kFloat32 &&
              db.numel() == dl.size(1), "vocab head: dl bf16 [rows, C], db fp32 [C]");
  check(ts_vocab_head_colsum(dl.data_ptr(), db.data_ptr<float>(), (int)dl.size(0), (int)dl.size(1), accumulate ? 1 : 0, stream()),
        "vocab_head_colsum");
}

// ---- sampling the next token (csrc/head_vocab.cu) -------------------------------------------------------------------
// tokens int32 [B] (written), step int32 [1] (read, advanced by one), row0 int32 [1] (the noise counter's row word of row 0),
// optional rec_tok int32 / rec_lp fp32 [B, N] (column
// step - s0 written) -> logprob fp32 [B].  Scratch is allocated here; nothing is read back to the host.
struct SampleOut {
  int* rec_tok = nullptr;
  float* rec_lp = nullptr;
  int N = 0;
};
SampleOut sample_check(int64_t B, const Tensor& like, const Tensor& step, const Tensor& row0, const Tensor& tokens,
                       const std::optional<Tensor>& rec_tok, const std::optional<Tensor>& rec_lp, double temperature) {
  chk_cuda(step, "step"); chk_cuda(row0, "row0"); chk_cuda(tokens, "tokens");
  TORCH_CHECK(row0.scalar_type() == torch::kInt32 && row0.numel() == 1 && row0.device() == like.device(), "vocab sample: row0 int32 [1]");
  TORCH_CHECK(std::isfinite(temperature) && temperature >= 0, "vocab sample: temperature must be finite and >= 0");
  TORCH_CHECK(step.scalar_type() == torch::kInt32 && step.numel() == 1 && step.device() == like.device(), "vocab sample: step int32 [1]");
  TORCH_CHECK(tokens.scalar_type() == torch::kInt32 && tokens.numel() == B && tokens.device() == like.device(), "vocab sample: tokens int32 [B]");
  SampleOut o;
  TORCH_CHECK(rec_tok.has_value() == rec_lp.has_value(), "vocab sample: rec_tok and rec_lp go together");
  if (rec_tok.has_value()) {
    chk_cuda(*rec_tok, "rec_tok"); chk_cuda(*rec_lp, "rec_lp");
    TORCH_CHECK(rec_tok->scalar_type() == torch::kInt32 && rec_tok->dim() == 2 && rec_tok->size(0) == B &&
                rec_lp->scalar_type() == torch::kFloat32 && rec_lp->sizes() == rec_tok->sizes() &&
                rec_tok->device() == like.device() && rec_lp->device() == like.device(), "vocab sample: records int32 / fp32 [B, N]");
    o.rec_tok = rec_tok->data_ptr<int>(); o.rec_lp = rec_lp->data_ptr<float>(); o.N = (int)rec_tok->size(1);
  }
  return o;
}

Tensor vocab_sample(const Tensor& h, const Tensor& Wb, bool w_kmajor, const Tensor& bias, double temperature, int64_t seed, Tensor step,
                    const Tensor& row0, Tensor tokens, const std::optional<Tensor>& rec_tok, const std::optional<Tensor>& rec_lp,
                    int64_t s0) {
  chk_cuda(h, "h"); chk_cuda(Wb, "Wb"); chk_cuda(bias, "bias");
  const int64_t Cw = vocab_classes(h, Wb, w_kmajor, "vocab sample");
  TORCH_CHECK(h.size(0) >= 1 && h.size(0) < (int64_t(1) << 24), "vocab sample: h bf16 [B,H] with 1 <= B < 2^24");
  TORCH_CHECK(h.size(1) % 64 == 0 && Cw % 8 == 0 && Cw >= 8, "vocab sample: H % 64 == 0 and C % 8 == 0");
  TORCH_CHECK(bias.scalar_type() == torch::kFloat32 && bias.numel() == Cw && ((uintptr_t)bias.data_ptr() % 8) == 0,
              "vocab sample: bias fp32 [C]");
  c10::cuda::CUDAGuard g(h.device());
  const int B = h.size(0), H = h.size(1), C = (int)Cw;
  const SampleOut o = sample_check(B, h, step, row0, tokens, rec_tok, rec_lp, temperature);
  const int nt = ts_vocab_head_parts(C);
  auto fo = torch::TensorOptions().device(h.device()).dtype(torch::kFloat32);
  auto part = torch::empty({(int64_t)B * nt * 4}, fo), logprob = torch::empty({B}, fo);
  auto part_arg = torch::empty({(int64_t)B * nt}, fo.dtype(torch::kInt32)), ticket = torch::zeros({1}, fo.dtype(torch::kInt32));
  check(ts_vocab_sample(h.data_ptr(), Wb.data_ptr(), w_kmajor ? 1 : 0, bias.data_ptr<float>(), (float)temperature, (unsigned int)(seed & 0xffffffff),
                        step.data_ptr<int>(), row0.data_ptr<int>(), part.data_ptr(), part_arg.data_ptr<int>(), (unsigned int*)ticket.data_ptr<int>(),
                        tokens.data_ptr<int>(), logprob.data_ptr<float>(), o.rec_tok, o.rec_lp, o.N, (int)s0, B, H, C, h.get_device(),
                        stream()), "vocab_sample");
  return logprob;
}

void chk_logits(const Tensor& logits) {
  chk_cuda(logits, "logits");
  TORCH_CHECK(logits.dim() == 2 && logits.scalar_type() == torch::kFloat32 && logits.is_contiguous() && logits.size(0) >= 1 &&
              logits.size(1) >= 1 && logits.size(1) < (int64_t(1) << 31) && logits.numel() < (int64_t(1) << 40),
              "vocab sample: logits fp32 [B, C], packed");
}

// The same from fp32 logits [B, C] (bias included).  tau fp32 [B] (top-k / top-p, temperature > 0): only the classes with
// l >= tau[b] are candidates.
Tensor vocab_sample_logits(const Tensor& logits, double temperature, int64_t seed, Tensor step, const Tensor& row0, Tensor tokens,
                           const std::optional<Tensor>& rec_tok, const std::optional<Tensor>& rec_lp, int64_t s0,
                           const std::optional<Tensor>& tau) {
  chk_logits(logits);
  c10::cuda::CUDAGuard g(logits.device());
  const int B = logits.size(0), C = logits.size(1);
  const SampleOut o = sample_check(B, logits, step, row0, tokens, rec_tok, rec_lp, temperature);
  if (tau.has_value()) {
    chk_cuda(*tau, "tau");
    TORCH_CHECK(tau->scalar_type() == torch::kFloat32 && tau->numel() == B && tau->is_contiguous() && tau->device() == logits.device(),
                "vocab sample: tau fp32 [B]");
    TORCH_CHECK(temperature > 0, "vocab sample: a threshold needs temperature > 0 (greedy keeps the arg-max, which no filter drops)");
  }
  const int nt = ts_vocab_head_parts(C);
  auto fo = torch::TensorOptions().device(logits.device()).dtype(torch::kFloat32);
  auto part = torch::empty({(int64_t)B * nt * 4}, fo), logprob = torch::empty({B}, fo);
  auto part_arg = torch::empty({(int64_t)B * nt}, fo.dtype(torch::kInt32)), ticket = torch::zeros({1}, fo.dtype(torch::kInt32));
  check(ts_vocab_sample_logits(logits.data_ptr<float>(), tau.has_value() ? tau->data_ptr<float>() : nullptr, (float)temperature,
                               (unsigned int)(seed & 0xffffffff), step.data_ptr<int>(),
                               row0.data_ptr<int>(), part.data_ptr(), part_arg.data_ptr<int>(), (unsigned int*)ticket.data_ptr<int>(), tokens.data_ptr<int>(),
                               logprob.data_ptr<float>(), o.rec_tok, o.rec_lp, o.N, (int)s0, B, C, stream()), "vocab_sample_logits");
  return logprob;
}

// logits fp32 [B, C] = h W + bias from the sampling kernel's main loop: the values vocab_sample scores, stored (top-k / top-p).
Tensor vocab_head_logits(const Tensor& h, const Tensor& Wb, bool w_kmajor, const Tensor& bias) {
  chk_cuda(h, "h"); chk_cuda(Wb, "Wb"); chk_cuda(bias, "bias");
  const int64_t Cw = vocab_classes(h, Wb, w_kmajor, "vocab logits");
  TORCH_CHECK(h.is_contiguous() && h.size(0) >= 1 && h.size(0) < (int64_t(1) << 24), "vocab logits: h bf16 [B,H] packed, 1 <= B < 2^24");
  TORCH_CHECK(h.size(1) % 64 == 0 && Cw % 8 == 0 && Cw >= 8, "vocab logits: H % 64 == 0 and C % 8 == 0");
  TORCH_CHECK(bias.scalar_type() == torch::kFloat32 && bias.numel() == Cw && ((uintptr_t)bias.data_ptr() % 8) == 0,
              "vocab logits: bias fp32 [C]");
  c10::cuda::CUDAGuard g(h.device());
  const int B = h.size(0), H = h.size(1), C = (int)Cw;
  auto logits = torch::empty({B, C}, torch::TensorOptions().device(h.device()).dtype(torch::kFloat32));
  check(ts_vocab_head_logits(h.data_ptr(), Wb.data_ptr(), w_kmajor ? 1 : 0, bias.data_ptr<float>(), logits.data_ptr<float>(), B, H, C,
                             h.get_device(), stream()), "vocab_head_logits");
  return logits;
}

// tau fp32 [B]: the top-k / top-p threshold of each row of logits fp32 [B, C] (csrc/head_vocab.cu, vocab_threshold_kernel);
// top_k 0 and top_p 1 are off.  No host sync: the filters are kernel arguments.
Tensor vocab_threshold(const Tensor& logits, int64_t top_k, double top_p, double temperature) {
  chk_logits(logits);
  TORCH_CHECK(top_k >= 0, "vocab threshold: top_k must be >= 0 (0 = off), got ", top_k);
  TORCH_CHECK(std::isfinite(top_p) && top_p > 0 && top_p <= 1, "vocab threshold: top_p must be in (0, 1] (1 = off), got ", top_p);
  TORCH_CHECK(std::isfinite(temperature) && temperature > 0, "vocab threshold: temperature must be finite and > 0, got ", temperature);
  c10::cuda::CUDAGuard g(logits.device());
  const int B = logits.size(0), C = logits.size(1);
  auto tau = torch::empty({B}, torch::TensorOptions().device(logits.device()).dtype(torch::kFloat32));
  check(ts_vocab_threshold(logits.data_ptr<float>(), B, C, (int)std::min<int64_t>(top_k, C), top_p, (float)temperature,
                           tau.data_ptr<float>(), stream()), "vocab_threshold");
  return tau;
}

// ---- pooling over time (csrc/seq_pool.cu) ---------------------------------------------------------------------
// h: the top layer's h_seq as contiguous [T·B, H] time-major rows (bf16 or fp32); mode 0 mean, 1 max, 2 attention.
void chk_f32(const Tensor& t, int64_t numel, const char* n) {
  chk_cuda(t, n);
  TORCH_CHECK(t.scalar_type() == torch::kFloat32 && t.numel() == numel, n, ": fp32 with ", numel, " elements");
}

// -> (s fp32 [B,H], argmax int32 [B,H] (max; else empty)); alpha fp32 [T,B] for attention.
std::vector<Tensor> seq_pool_fwd(const Tensor& h, const std::optional<Tensor>& lengths, int64_t T, int64_t mode,
                                 const std::optional<Tensor>& alpha) {
  chk_cuda(h, "h");
  TORCH_CHECK(h.dim() == 2 && T >= 1 && h.size(0) % T == 0, "seq_pool_fwd: h [T·B, H]");
  TORCH_CHECK(mode >= 0 && mode <= 2, "seq_pool_fwd: mode 0 mean, 1 max, 2 attention");
  c10::cuda::CUDAGuard g(h.device());
  const int B = h.size(0) / T, H = h.size(1);
  if (mode == 2) {
    TORCH_CHECK(alpha.has_value(), "seq_pool_fwd: attention needs alpha");
    chk_f32(*alpha, (int64_t)T * B, "alpha");
  }
  auto fo = h.options().dtype(torch::kFloat32);
  auto s = torch::empty({B, H}, fo);
  auto am = mode == 1 ? torch::empty({B, H}, fo.dtype(torch::kInt32)) : torch::empty({0}, fo.dtype(torch::kInt32));
  check(ts_seq_pool_fwd(h.data_ptr(), is_bf16(h), lengths_ptr(lengths, B, h), fptr(alpha), (int)mode, (int)T, B, H,
                        s.data_ptr<float>(), mode == 1 ? am.data_ptr<int>() : nullptr, stream()), "seq_pool_fwd");
  return {s, am};
}

// u fp32 [T·B, A]: h W_a in, tanh(h W_a + b_a) out (0 at uncounted steps) -> alpha fp32 [T,B], the softmax over counted steps.
// exact: tanh in fp64 rounded once (fp32 h), else tanh.approx (bf16 h).
Tensor seq_pool_attn_scores(Tensor u, const Tensor& ba, const Tensor& v, const std::optional<Tensor>& lengths, int64_t T, bool exact) {
  chk_cuda(u, "u");
  TORCH_CHECK(u.dim() == 2 && u.scalar_type() == torch::kFloat32 && T >= 1 && u.size(0) % T == 0, "seq_pool_attn_scores: u fp32 [T·B, A]");
  c10::cuda::CUDAGuard g(u.device());
  const int B = u.size(0) / T, A = u.size(1);
  chk_f32(ba, A, "b_a"); chk_f32(v, A, "v");
  auto alpha = torch::empty({T, B}, u.options());
  check(ts_seq_pool_attn_scores(u.data_ptr<float>(), ba.data_ptr<float>(), v.data_ptr<float>(), lengths_ptr(lengths, B, u), (int)T, B, A,
                                alpha.data_ptr<float>(), (int)exact, stream()), "seq_pool_attn_scores");
  return alpha;
}

// -> dU [T·B, A] (dtype of h; 0 at uncounted steps); dv, dba fp32 [A] written (or accumulated into, acc_*) in a fixed order.
Tensor seq_pool_attn_bwd(const Tensor& h, const Tensor& ds, const Tensor& alpha, const Tensor& u, const Tensor& v,
                         const std::optional<Tensor>& lengths, int64_t T, Tensor dv, Tensor dba, bool acc_dv, bool acc_dba) {
  chk_cuda(h, "h");
  TORCH_CHECK(h.dim() == 2 && T >= 1 && h.size(0) % T == 0, "seq_pool_attn_bwd: h [T·B, H]");
  c10::cuda::CUDAGuard g(h.device());
  const int B = h.size(0) / T, H = h.size(1), A = u.size(1);
  chk_f32(ds, (int64_t)B * H, "ds"); chk_f32(alpha, (int64_t)T * B, "alpha"); chk_f32(u, (int64_t)T * B * A, "u");
  chk_f32(v, A, "v"); chk_f32(dv, A, "dv"); chk_f32(dba, A, "dba");
  auto fo = h.options().dtype(torch::kFloat32);
  auto dU = torch::empty({h.size(0), A}, h.options());
  auto dalpha = torch::empty({T, B}, fo);
  auto partial = torch::empty({B, 2 * A}, fo);
  auto ticket = torch::zeros({1}, fo.dtype(torch::kInt32));
  check(ts_seq_pool_attn_bwd(h.data_ptr(), is_bf16(h), ds.data_ptr<float>(), alpha.data_ptr<float>(), u.data_ptr<float>(),
                             v.data_ptr<float>(), lengths_ptr(lengths, B, h), (int)T, B, H, A, dalpha.data_ptr<float>(), dU.data_ptr(),
                             partial.data_ptr<float>(), (unsigned int*)ticket.data_ptr<int>(), dv.data_ptr<float>(), dba.data_ptr<float>(),
                             acc_dv ? 1 : 0, acc_dba ? 1 : 0, stream()), "seq_pool_attn_bwd");
  return dU;
}

// ds fp32 [B,H] -> dh_seq [T·B, H] (bf16 when out_bf16, else fp32), 0 at uncounted steps.  max: argmax int32 [B,H];
// attention: alpha fp32 [T,B] and G = dU W_a^T fp32 [T·B, H] (added before the one rounding).
Tensor seq_pool_bwd(const Tensor& ds, const std::optional<Tensor>& lengths, int64_t T, int64_t mode, const std::optional<Tensor>& argmax,
                    const std::optional<Tensor>& alpha, const std::optional<Tensor>& G, bool out_bf16) {
  chk_cuda(ds, "ds");
  TORCH_CHECK(ds.dim() == 2 && ds.scalar_type() == torch::kFloat32 && T >= 1, "seq_pool_bwd: ds fp32 [B,H]");
  TORCH_CHECK(mode >= 0 && mode <= 2, "seq_pool_bwd: mode 0 mean, 1 max, 2 attention");
  c10::cuda::CUDAGuard g(ds.device());
  const int B = ds.size(0), H = ds.size(1);
  if (mode == 1) {
    TORCH_CHECK(argmax.has_value() && argmax->scalar_type() == torch::kInt32 && argmax->numel() == (int64_t)B * H, "seq_pool_bwd: argmax int32 [B,H]");
    chk_cuda(*argmax, "argmax");
  }
  if (mode == 2) {
    TORCH_CHECK(alpha.has_value() && G.has_value(), "seq_pool_bwd: attention needs alpha and G");
    chk_f32(*alpha, (int64_t)T * B, "alpha"); chk_f32(*G, (int64_t)T * B * H, "G");
  }
  auto dh = torch::empty({T * B, H}, ds.options().dtype(out_bf16 ? torch::kBFloat16 : torch::kFloat32));
  check(ts_seq_pool_bwd(ds.data_ptr<float>(), lengths_ptr(lengths, B, ds), mode == 1 ? argmax->data_ptr<int>() : nullptr, fptr(alpha),
                        fptr(G), (int)mode, (int)T, B, H, dh.data_ptr(), out_bf16 ? 1 : 0, stream()), "seq_pool_bwd");
  return dh;
}

// ---- token embedding (csrc/embedding.cu) ------------------------------------------------------------------------
void chk_tokens(const Tensor& tok, const Tensor& like) {
  chk_cuda(tok, "tokens");
  TORCH_CHECK(tok.device() == like.device() && tok.scalar_type() == torch::kInt32 && tok.dim() == 2,
              "tokens must be int32 [B,T] on the table's device");
}

// table [V,E] (bf16 or fp32), tokens int32 [B,T] -> x [T,B,E] of the table's dtype, time-major.  in_step / in_desc: input
// dropout over each position's E units, row_step / row_desc: embedding dropout over the V rows (drop_args; None = off).
Tensor embed_fwd(const Tensor& table, const Tensor& tokens, const std::optional<Tensor>& lengths,
                 const std::optional<Tensor>& in_step, const std::vector<int64_t>& in_desc,
                 const std::optional<Tensor>& row_step, const std::vector<int64_t>& row_desc) {
  chk_cuda(table, "table");
  TORCH_CHECK(table.dim() == 2, "embed_fwd: table [V,E]");
  chk_tokens(tokens, table);
  c10::cuda::CUDAGuard g(table.device());
  const int B = tokens.size(0), T = tokens.size(1), V = table.size(0), E = table.size(1);
  auto x = torch::empty({T, B, E}, table.options());
  unsigned int di[5], de[5];
  const int* is = drop_args(in_step, in_desc, table, di);
  const int* rs = drop_args(row_step, row_desc, table, de);
  check(ts_embed_fwd(table.data_ptr(), is_bf16(table), tokens.data_ptr<int>(), lengths_ptr(lengths, B, table), T, B, E, V,
                     x.data_ptr(), is, di, rs, de, stream()), "embed_fwd");
  return x;
}

// Per-device scratch of the backward pass: {zeroed (2 V int32 words that are zero between calls, the kernels restore them),
// working ints, partial floats}.  A buffer only grows, and a replaced one is kept alive: a captured graph holds its pointers.
struct EmbedScratch { int* zeroed; int* ints; float* floats; };
EmbedScratch embed_scratch(const Tensor& like, int64_t N, int64_t V, int64_t E) {
  static std::vector<std::vector<Tensor>> bufs(64, std::vector<Tensor>(3));
  static std::vector<Tensor> retired;
  auto& b = bufs[like.device().index()];
  long long need[2];
  ts_embed_scratch_numel(N, V, E, need);
  const int64_t sizes[3] = {2 * V, need[0], need[1]};
  for (int i = 0; i < 3; ++i) {
    if (b[i].defined() && b[i].numel() >= sizes[i]) continue;
    if (b[i].defined()) retired.push_back(b[i]);
    auto opt = torch::TensorOptions().device(like.device()).dtype(i == 2 ? torch::kFloat32 : torch::kInt32);
    b[i] = i == 0 ? torch::zeros({sizes[i]}, opt) : torch::empty({sizes[i]}, opt);
  }
  return {b[0].data_ptr<int>(), b[1].data_ptr<int>(), b[2].data_ptr<float>()};
}

// dx [T·B, E] (bf16 or fp32) -> dW fp32 [V,E]: every row written (accumulate false) or added to the rows of ids present; the
// dropout arguments are the forward's (embed_fwd)
void embed_bwd(const Tensor& dx, const Tensor& tokens, const std::optional<Tensor>& lengths, Tensor dW, bool accumulate,
               const std::optional<Tensor>& in_step, const std::vector<int64_t>& in_desc,
               const std::optional<Tensor>& row_step, const std::vector<int64_t>& row_desc) {
  chk_cuda(dx, "dx"); chk_cuda(dW, "dW");
  chk_tokens(tokens, dx);
  const int B = tokens.size(0), T = tokens.size(1);
  TORCH_CHECK(dW.dim() == 2 && dW.scalar_type() == torch::kFloat32 && dW.device() == dx.device(), "embed_bwd: dW fp32 [V,E]");
  const int V = dW.size(0), E = dW.size(1);
  TORCH_CHECK(dx.numel() == (int64_t)T * B * E, "embed_bwd: dx [T·B, E]");
  c10::cuda::CUDAGuard g(dx.device());
  unsigned int di[5], de[5];
  const int* is = drop_args(in_step, in_desc, dx, di);
  const int* rs = drop_args(row_step, row_desc, dx, de);
  auto s = embed_scratch(dx, (int64_t)T * B, V, E);
  check(ts_embed_bwd(dx.data_ptr(), is_bf16(dx), tokens.data_ptr<int>(), lengths_ptr(lengths, B, dx), T, B, E, V,
                     dW.data_ptr<float>(), accumulate ? 1 : 0, s.zeroed, s.ints, s.floats, is, di, rs, de, stream()), "embed_bwd");
}

// ---- optimizer ----------------------------------------------------------------------------------------------
// clip: the fp32 [2] {norm, coef} flat_grad_norm wrote on this stream; the update then uses coef * g_total.
const float* clip_ptr(const std::optional<Tensor>& clip, const Tensor& p) {
  if (!clip.has_value()) return nullptr;
  TORCH_CHECK(clip->is_cuda() && clip->device() == p.device() && clip->scalar_type() == torch::kFloat32 && clip->numel() == 2 &&
              clip->is_contiguous(), "clip must be a contiguous fp32 [2] tensor on p's device (flat_grad_norm's out)");
  return clip->data_ptr<float>();
}
void flat_adam(Tensor p, const Tensor& g, Tensor m, Tensor v, std::optional<Tensor> shadow, double lr_t, double b1,
               double b2, double eps, double wd, double gscale, std::optional<Tensor> step_dev, int64_t wd_numel,
               std::optional<Tensor> clip) {
  chk_cuda(p, "p"); chk_cuda(g, "g"); chk_cuda(m, "m"); chk_cuda(v, "v");
  c10::cuda::CUDAGuard gd(p.device());
  TORCH_CHECK(p.numel() == g.numel() && p.numel() == m.numel() && p.numel() == v.numel(), "numel mismatch");
  check(ts_flat_adam(p.data_ptr<float>(), g.data_ptr<float>(), m.data_ptr<float>(), v.data_ptr<float>(),
                     shadow.has_value() ? shadow->data_ptr() : nullptr, p.numel(), lr_t, b1, b2, eps, wd, gscale, stream(),
                     step_dev.has_value() ? step_dev->data_ptr<int>() : nullptr, (long long)wd_numel, clip_ptr(clip, p)),
        "flat_adam");
}
void flat_sgd(Tensor p, const Tensor& g, std::optional<Tensor> shadow, double lr, double wd, double gscale, int64_t wd_numel,
              std::optional<Tensor> clip) {
  chk_cuda(p, "p"); chk_cuda(g, "g");
  c10::cuda::CUDAGuard gd(p.device());
  check(ts_flat_sgd(p.data_ptr<float>(), g.data_ptr<float>(), shadow.has_value() ? shadow->data_ptr() : nullptr,
                    p.numel(), lr, wd, gscale, stream(), (long long)wd_numel, clip_ptr(clip, p)), "flat_sgd");
}
// out = {||g_total||_2, min(max_norm / (norm + 1e-6), 1)} with g_total = g * gscale + wd * p over [0, wd_numel) (-1: all) and
// g * gscale beyond; scratch: float64 [flat_grad_norm_scratch(n)], zeroed before its first use (each call leaves its ticket 0).
void flat_grad_norm(const Tensor& g, const Tensor& p, Tensor out, Tensor scratch, double max_norm, double wd, double gscale,
                    int64_t wd_numel) {
  chk_cuda(g, "g"); chk_cuda(p, "p"); chk_cuda(out, "out"); chk_cuda(scratch, "scratch");
  c10::cuda::CUDAGuard gd(g.device());
  TORCH_CHECK(g.scalar_type() == torch::kFloat32 && p.scalar_type() == torch::kFloat32 && p.numel() == g.numel(), "flat_grad_norm: g, p fp32 of one size");
  TORCH_CHECK(out.scalar_type() == torch::kFloat32 && out.numel() == 2, "flat_grad_norm: out fp32 [2]");
  TORCH_CHECK(scratch.scalar_type() == torch::kFloat64 && scratch.numel() >= ts_flat_grad_norm_scratch(g.numel()),
              "flat_grad_norm: scratch float64 [flat_grad_norm_scratch(n)]");
  TORCH_CHECK(p.device() == g.device() && out.device() == g.device() && scratch.device() == g.device(), "flat_grad_norm: one device");
  check(ts_flat_grad_norm(g.data_ptr<float>(), p.data_ptr<float>(), g.numel(), wd, gscale, (long long)wd_numel, max_norm,
                          scratch.data_ptr<double>(), out.data_ptr<float>(), stream()), "flat_grad_norm");
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
// rowsum: optional fp32 [M] that also receives the row sums of op(A) over K (overwritten, or accumulated with rowsum_acc).
Tensor gemm2(const Tensor& A, const Tensor& B, const std::optional<Tensor>& bias, std::optional<Tensor> out, bool a_mn, bool b_mn,
             bool out_fp32, bool accumulate, int64_t ctas, int64_t bn, int64_t max_ctas, const std::optional<Tensor>& gate,
             const std::vector<int64_t>& gate_cfg, const std::optional<Tensor>& done, const std::optional<Tensor>& gate_err,
             int64_t stream_handle, bool pdl, int64_t a_fold, int64_t b_fold, int64_t fold_cols, const std::optional<Tensor>& rowsum,
             bool rowsum_acc) {
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
  float* rp = nullptr;
  if (rowsum.has_value()) {
    TORCH_CHECK(rowsum->is_cuda() && rowsum->scalar_type() == torch::kFloat32 && rowsum->is_contiguous() && rowsum->numel() == M &&
                C.scalar_type() == torch::kFloat32, "gemm2: rowsum must be a contiguous fp32 [M] next to an fp32 output");
    rp = rowsum->data_ptr<float>();
  }
  TORCH_CHECK((ctas == 1 || ctas == 2) && (bn == 128 || bn == 256), "gemm2: ctas must be 1 or 2 and bn 128 or 256 (got ", ctas, ", ", bn, ")");
  unsigned int* dp = nullptr;
  if (done.has_value()) {
    TORCH_CHECK(done->is_cuda() && done->scalar_type() == torch::kInt32 && done->is_contiguous(), "gemm2: done must be a contiguous int32 cuda tensor");
    // one counter per 128-row block and bn-column tile; a 2-CTA cluster's peer counts its block even where all its rows lie past M
    const int64_t blocks = (M + 128 * ctas - 1) / (128 * ctas) * ctas * ((N + bn - 1) / bn);
    TORCH_CHECK(done->numel() >= blocks, "gemm2: done needs ceil(M / (128 * ctas)) * ctas * ceil(N / bn) = ", blocks,
                " counters, got ", done->numel());
    dp = (unsigned int*)done->data_ptr<int>();
  }
  check(ts_gemm2(A.data_ptr(), B.data_ptr(), C.data_ptr(), fptr(bias), M, N, K, (int)A.stride(0), (int)B.stride(0), (int)C.stride(0),
                 a_mn ? 1 : 0, b_mn ? 1 : 0, out_mode, (int)ctas, (int)bn, A.device().index(), (int)max_ctas, gp, gcfg, dp,
                 gate_err.has_value() ? gate_err->data_ptr<int>() : nullptr, pdl ? 1 : 0, (int)a_fold, (int)b_fold, (int)fold_cols,
                 rp, rowsum_acc ? 1 : 0, stream_handle ? (cudaStream_t)stream_handle : stream()), "gemm2");
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
  m.def("seq_pool_fwd", &seq_pool_fwd, py::arg("h"), py::arg("lengths"), py::arg("T"), py::arg("mode"), py::arg("alpha"));
  m.def("seq_pool_attn_scores", &seq_pool_attn_scores, py::arg("u"), py::arg("b_a"), py::arg("v"), py::arg("lengths"), py::arg("T"),
        py::arg("exact") = false);
  m.def("seq_pool_attn_bwd", &seq_pool_attn_bwd, py::arg("h"), py::arg("ds"), py::arg("alpha"), py::arg("u"), py::arg("v"),
        py::arg("lengths"), py::arg("T"), py::arg("dv"), py::arg("dba"), py::arg("acc_dv"), py::arg("acc_dba"));
  m.def("seq_pool_bwd", &seq_pool_bwd, py::arg("ds"), py::arg("lengths"), py::arg("T"), py::arg("mode"), py::arg("argmax"),
        py::arg("alpha"), py::arg("G"), py::arg("out_bf16"));
  m.def("embed_fwd", &embed_fwd, py::arg("table"), py::arg("tokens"), py::arg("lengths"), py::arg("in_step") = py::none(),
        py::arg("in_desc") = std::vector<int64_t>{}, py::arg("row_step") = py::none(), py::arg("row_desc") = std::vector<int64_t>{});
  m.def("embed_bwd", &embed_bwd, py::arg("dx"), py::arg("tokens"), py::arg("lengths"), py::arg("dW"), py::arg("accumulate"),
        py::arg("in_step") = py::none(), py::arg("in_desc") = std::vector<int64_t>{}, py::arg("row_step") = py::none(),
        py::arg("row_desc") = std::vector<int64_t>{});
  m.attr("EMBED_BWD_LAUNCHES") = ts_embed_bwd_launches();
  m.def("head_step_fwd", &head_step_fwd, py::arg("h"), py::arg("W"), py::arg("bias"), py::arg("labels"), py::arg("lengths"), py::arg("T"));
  m.def("head_step_bwd", &head_step_bwd, py::arg("h"), py::arg("W"), py::arg("dlogits"), py::arg("dloss"), py::arg("dW"), py::arg("db"),
        py::arg("acc_w"), py::arg("acc_b"));
  m.def("vocab_head_parts", [](int64_t C) { return ts_vocab_head_parts((int)C); });
  m.def("vocab_head_fwd", &vocab_head_fwd, py::arg("h"), py::arg("Wb"), py::arg("w_kmajor"), py::arg("bias"), py::arg("labels"), py::arg("lengths"),
        py::arg("T"), py::arg("part"));
  m.def("vocab_head_dlogits", &vocab_head_dlogits, py::arg("h"), py::arg("Wb"), py::arg("w_kmajor"), py::arg("bias"), py::arg("labels"), py::arg("lengths"),
        py::arg("T"), py::arg("lse"), py::arg("count"), py::arg("dloss"), py::arg("row0"), py::arg("rows"), py::arg("dl"));
  m.def("vocab_head_colsum", &vocab_head_colsum, py::arg("dl"), py::arg("db"), py::arg("accumulate"));
  m.def("vocab_sample", &vocab_sample, py::arg("h"), py::arg("Wb"), py::arg("w_kmajor"), py::arg("bias"), py::arg("temperature"), py::arg("seed"),
        py::arg("step"), py::arg("row0"), py::arg("tokens"), py::arg("rec_tok"), py::arg("rec_lp"), py::arg("s0"));
  m.def("vocab_sample_logits", &vocab_sample_logits, py::arg("logits"), py::arg("temperature"), py::arg("seed"), py::arg("step"),
        py::arg("row0"), py::arg("tokens"), py::arg("rec_tok"), py::arg("rec_lp"), py::arg("s0"), py::arg("tau") = py::none());
  m.def("vocab_head_logits", &vocab_head_logits, py::arg("h"), py::arg("Wb"), py::arg("w_kmajor"), py::arg("bias"));
  m.def("vocab_threshold", &vocab_threshold, py::arg("logits"), py::arg("top_k"), py::arg("top_p"), py::arg("temperature"));
  m.def("head_bwd", &head_bwd, py::arg("h"), py::arg("W"), py::arg("dlogits"), py::arg("dloss"), py::arg("dW"), py::arg("db"),
        py::arg("acc_w") = false, py::arg("acc_b") = false);
  m.def("flat_adam", &flat_adam, py::arg("p"), py::arg("g"), py::arg("m"), py::arg("v"), py::arg("shadow"), py::arg("lr_t"),
        py::arg("b1"), py::arg("b2"), py::arg("eps"), py::arg("wd"), py::arg("gscale"), py::arg("step_dev") = py::none(),
        py::arg("wd_numel") = -1, py::arg("clip") = py::none());
  m.def("flat_sgd", &flat_sgd, py::arg("p"), py::arg("g"), py::arg("shadow"), py::arg("lr"), py::arg("wd"), py::arg("gscale"),
        py::arg("wd_numel") = -1, py::arg("clip") = py::none());
  m.def("flat_grad_norm", &flat_grad_norm, py::arg("g"), py::arg("p"), py::arg("out"), py::arg("scratch"), py::arg("max_norm"),
        py::arg("wd") = 0.0, py::arg("gscale") = 1.0, py::arg("wd_numel") = -1);
  m.def("flat_grad_norm_scratch", [](int64_t n) { return ts_flat_grad_norm_scratch((long long)n); });
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
        py::arg("fold_cols") = 0, py::arg("rowsum") = py::none(), py::arg("rowsum_acc") = false);
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
  m.def("weight_drop_grad", &weight_drop_grad, py::arg("src"), py::arg("dst"), py::arg("step"), py::arg("desc"),
        py::arg("accumulate") = false);
}
