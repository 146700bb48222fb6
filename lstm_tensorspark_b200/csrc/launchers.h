// The C interface of the kernel launchers that bindings.cpp calls, declared once.  The .cu file that defines a launcher
// includes this header too, so a definition whose parameters differ from its declaration fails to compile (a C-linkage
// symbol carries no parameter types: the linker would accept the mismatch).  Grouped by defining file, in that file's order.
// Compiled by g++ (bindings.cpp) and nvcc (the .cu files): CUDA runtime types only.
#pragma once
#include <cuda_runtime.h>

extern "C" {

// activation_reg.cu
long long ts_act_reg_scratch(int T, int B, int H, int is_bf16);
int ts_act_reg_fwd(const void* out, const void* h, const int* lengths, int T, int B, int H, int is_bf16, double* scratch, float* sums,
                   cudaStream_t st);
int ts_act_reg_bwd(const void* dh, const void* out, const void* h, const int* lengths, const float* g, int T, int B, int H, int is_bf16,
                   const int* drop_step, const unsigned int* drop_desc, void* dst, cudaStream_t st);
// cache_pointer.cu
int ts_cache_key_tile();
int ts_cache_chunks(int T, int B, int H, int W);
int ts_cache_combine_blocks(int R);
int ts_cache_pointer(const void* h, const void* keys, const int* klab, const long long* labels, const float* logp_model, const int* lengths,
                     int T, int B, int H, int W, int Cap, long long P0, float theta, float lambda, int bf16, int tc, void* part,
                     void* block_sums, unsigned int* ticket, float* logp, float* sums, cudaStream_t st);
int ts_cache_append(const void* h, void* keys, int* klab, const long long* labels, int T, int B, long long row_bytes, int Cap, long long P0,
                    cudaStream_t st);
int ts_cache_label_logprob_parts(const void* part, const float* lse, const long long* labels, float* logp, int T, int B, int C, int nt,
                                 cudaStream_t st);
int ts_cache_label_logprob_logits(const float* logits, const long long* labels, float* logp, int T, int B, int C, cudaStream_t st);
// embedding.cu
void ts_embed_scratch_numel(long long N, long long V, long long E, long long* ints);
int ts_embed_fwd(const void* table, int bf16, const int* tok, const int* lengths, int T, int B, int E, int V, void* x, const int* in_step,
                 const unsigned int* in_desc, const int* row_step, const unsigned int* row_desc, cudaStream_t st);
int ts_embed_bwd(const void* dx, int dx_bf16, const int* tok, const int* lengths, int T, int B, int E, int V, float* dW, int accumulate,
                 int* zeroed, int* scratch, float* partial, const int* in_step, const unsigned int* in_desc, const int* row_step,
                 const unsigned int* row_desc, cudaStream_t st);
int ts_embed_bwd_launches();
// fused_allreduce.cu
int ts_fused_allreduce(const unsigned long long* ptrs, unsigned long long mc_in, unsigned long long mc_param, unsigned long long mc_shadow,
                       float* m, float* v, unsigned int* epochs, int* err, long long n, int rank, int world, int mode, int two_shot,
                       int multicast, int blocks, float lr, float b1, float b2, float eps, float wd, double timeout_s, cudaStream_t st,
                       int* step_dev, long long wd_n, int bump_step, int pdl);
int ts_ar_bump_step(int* step_dev, cudaStream_t st);
int ts_ar_max_blocks();
int ts_ar_flag_words();
int ts_ar_slots();
// gemm2_wgmma.cu
int ts_gemm2(const void* A, const void* B, void* C, const float* bias, int M, int N, int K, int lda, int ldb, int ldc, int a_mn, int b_mn,
             int out_mode, int ctas, int bn, int dev, int max_ctas, const unsigned int* gate, const int* gate_cfg, unsigned int* done,
             int* gate_err, int pdl, int a_fold, int b_fold, int fold_cols, float* rowsum, int rowsum_acc, cudaStream_t st);
// gemm_generic.cu
int ts_gemm_generic(const void* A, const void* B, void* C, const float* bias, int M, int N, int K, long long a_rs, long long a_cs,
                    long long b_rs, long long b_cs, long long c_rs, int a_bf16, int b_bf16, int c_bf16, float beta, cudaStream_t st);
// head_vocab.cu
int ts_vocab_head_parts(int C);
int ts_vocab_head_blocks(int R);
int ts_vocab_head_fwd(const void* h, const void* Wb, int w_kmajor, const float* bias, const long long* labels, const int* lengths,
                      void* part, float* lse, float* part_loss, int* part_ok, unsigned int* ticket, float* loss, int* correct, int* count,
                      int T, int B, int H, int C, int dev, cudaStream_t st);
int ts_vocab_head_dlogits(const void* h, const void* Wb, int w_kmajor, const float* bias, const long long* labels, const int* lengths,
                          const float* lse, const float* dloss, const int* count, void* dl, int T, int B, int H, int C, int row0, int rows,
                          int dev, cudaStream_t st);
int ts_vocab_head_colsum(const void* dl, float* db, int rows, int C, int accumulate, cudaStream_t st);
int ts_vocab_sample(const void* h, const void* Wb, int w_kmajor, const float* bias, float temperature, unsigned int seed, int* step,
                    const int* row_base, void* part, int* part_arg, unsigned int* ticket, int* tokens, float* logprob, int* rec_tok,
                    float* rec_lp, int N, int s0, int B, int H, int C, int dev, cudaStream_t st);
int ts_vocab_sample_logits(const float* logits, const float* tau, float temperature, unsigned int seed, int* step, const int* row_base,
                           void* part, int* part_arg, unsigned int* ticket, int* tokens, float* logprob, int* rec_tok, float* rec_lp, int N,
                           int s0, int B, int C, cudaStream_t st);
int ts_vocab_head_logits(const void* h, const void* Wb, int w_kmajor, const float* bias, float* logits, int B, int H, int C, int dev,
                         cudaStream_t st);
int ts_vocab_threshold(const float* logits, int B, int C, int top_k, double top_p, float temperature, float* tau, cudaStream_t st);
// head_wgmma.cu
int ts_head_fwd_tc(const void* h, int ldh, const float* W, const float* bias, const long long* labels, float* logits, float* dlogits,
                   float* loss_sum, int* correct, int B, int H, int C, cudaStream_t st);
int ts_head_logits_generic(const void* h, const float* W, const float* bias, float* logits, int B, int H, int C, int is_bf16,
                           cudaStream_t st);
int ts_head_bwd(const void* h, const float* W, const float* dlogits, const float* dloss, void* dh, float* dW, float* db, int B, int H,
                int C, int is_bf16, int acc_w, int acc_b, cudaStream_t st);
int ts_head_step_fwd(const void* h, int ldh, int is_bf16, const float* W, const float* bias, const long long* labels, const int* lengths,
                     float* logits, float* dlogits, float* part_loss, int* part_ok, unsigned int* ticket, float* loss, int* correct,
                     int* count, int T, int B, int H, int C, int* used_tc, cudaStream_t st);
int ts_head_step_fwd_generic_parts(int R);
long long ts_head_step_bwd_scratch(int R, int H, int C);
int ts_head_step_bwd_tickets(int H);
int ts_head_step_bwd(const void* h, const float* W, const float* dlogits, const float* dloss, void* dh, float* dW, float* db,
                     float* scratch, unsigned int* tickets, int R, int H, int C, int is_bf16, int acc_w, int acc_b, cudaStream_t st);
// head_xent.cu
int ts_xent_rows(const float* logits, const long long* labels, float* dlogits, float* nll, float* loss_sum, int* correct, int B, int C,
                 int exact, cudaStream_t st);
// lstm_pointwise.cu
int ts_lstm_pointwise_fwd(const void* pre, const float* bias, const float* c_prev, void* h_out, float* c_out, void* act, int B, int H,
                          int is_bf16, cudaStream_t st, const void* h_prev, const int* lengths, int t);
int ts_lstm_pointwise_bwd(const void* dh_a, const float* dh_b, const float* dc_in, const void* act, const float* c_prev, const float* c_new,
                          void* dpre, float* dc_out, int B, int H, int is_bf16, cudaStream_t st, const int* lengths, int t, float* dh_out);
int ts_dropout(const void* x, void* y, int steps, int B, int H, int t0, int is_bf16, const int* drop_step, const unsigned int* drop_desc,
               cudaStream_t st);
int ts_weight_drop_grad(const float* src, float* dst, int R, int H, int accumulate, const int* drop_step, const unsigned int* drop_desc,
                        cudaStream_t st);
int ts_transpose01_rows(const void* src, void* dst, int B, int T, long long row_bytes, cudaStream_t st);
int ts_transpose2d_b16(const void* src, void* dst, int R, int C, cudaStream_t st);
long long ts_colsum_scratch_bytes(int rows, int cols);
int ts_colsum_bf16(const void* src, float* out, void* scratch, int rows, int cols, int pitch_cols, int accumulate, int pdl, int max_ctas,
                   cudaStream_t st);
// lstm_seq_wgmma.cu
int ts_lstm_seq_fwd(const void* gx, const void* w_h, const float* bias, const void* h_seq, const float* c_seq, void* act, const float* c0,
                    void* dbg, void* a_tiled, int T, int B, int H, unsigned int* sync_ws, int variant, cudaStream_t st, const void* h0,
                    const unsigned int* in_gate, int in_gate_tiles_n, int extra_signal, int launch_flags, const int* lengths, int reverse,
                    void* h_drop, const int* drop_step, const unsigned int* drop_desc);
int ts_lstm_seq_config(int bwd, int H, int B, int variant, int* out, int xchg_l2);
int ts_lstm_seq_prologue(const void* h0, const float* c0, void* h_seq, float* c_seq, void* a_tiled, unsigned int* sync_ws, int B, int H,
                         cudaStream_t st);
int ts_lstm_seq_bwd(const void* dh_seq, const void* w_hT, const void* act, const float* c_seq, const void* dpre, float* dh0, float* dc0,
                    void* dbg, void* a_tiled, int T, int B, int H, unsigned int* sync_ws, int variant, cudaStream_t st,
                    const unsigned int* in_gate, int in_gate_tiles_n, int extra_signal, int launch_flags, const int* lengths, int reverse,
                    const int* drop_step, const unsigned int* drop_desc, void* xchg);
int ts_lstm_seq_cluster_probe(int cluster);
// multi_tensor_opt.cu
int ts_flat_adam(float* p, const float* g, float* m, float* v, void* shadow, long long n, float lr_t, float b1, float b2, float eps,
                 float wd, float gscale, cudaStream_t st, int* step_dev, long long wd_n, const float* clip);
int ts_flat_sgd(float* p, const float* g, void* shadow, long long n, float lr, float wd, float gscale, cudaStream_t st, long long wd_n,
                const float* clip);
int ts_flat_asgd(float* p, const float* g, float* ax, int* avg, void* shadow, long long n, float lr, float wd, float gscale,
                 cudaStream_t st, long long wd_n, const float* clip);
int ts_flat_average(const float* p, float* ax, int* avg, long long n, cudaStream_t st);
int ts_flat_swap(float* p, float* ax, void* shadow, long long n, cudaStream_t st);
long long ts_flat_grad_norm_scratch(long long n);
int ts_flat_grad_norm(const float* g, const float* p, long long n, float wd, float gscale, long long wd_n, float max_norm, double* scratch,
                      float* out, cudaStream_t st);
int ts_cast_bf16(const float* p, void* shadow, long long n, cudaStream_t st);
// seq_pool.cu
int ts_seq_pool_fwd(const void* h, int h_bf16, const int* lengths, const float* alpha, int mode, int T, int B, int H, float* s, int* argmax,
                    cudaStream_t st);
int ts_seq_pool_attn_scores(float* u, const float* ba, const float* v, const int* lengths, int T, int B, int A, float* alpha, int exact,
                            cudaStream_t st);
int ts_seq_pool_attn_bwd(const void* h, int h_bf16, const float* ds, const float* alpha, const float* u, const float* v, const int* lengths,
                         int T, int B, int H, int A, float* dalpha, void* dU, float* partial, unsigned int* ticket, float* dv, float* dba,
                         int acc_dv, int acc_dba, cudaStream_t st);
int ts_seq_pool_bwd(const float* ds, const int* lengths, const int* argmax, const float* alpha, const float* G, int mode, int T, int B,
                    int H, void* dh, int out_bf16, cudaStream_t st);
// tmap.cu
const char* ts_last_error();

}  // extern "C"
