// t2_params.h — host-side parameter plumbing shared by the WaveNet, Tacotron and CBHG engines (defined in t2_params.cu):
// the flat parameter table, the fp32 -> bf16 operand pack jobs, the L2 regulariser, the workspace bump allocator and the side stream.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <initializer_list>
#include <string>
#include <vector>

namespace t2 {

inline long long align_up(long long v, long long a) { return (v + a - 1) / a * a; }
inline dim3 grid1d(long long n, int block = 256) { return dim3((unsigned)((n + block - 1) / block)); }

// 256-byte aligned bump allocator of the packed-operand and workspace byte offsets
struct Arena {
  long long used = 0;
  long long take(long long bytes) { const long long r = used; used = align_up(used + bytes, 256); return r; }
};

// one tensor of an engine's flat fp32 parameter buffer, in its TensorFlow variable layout
struct Param {
  std::string name;
  long long off;   // element offset in the flat buffer
  int ndim;
  int shape[4];    // unused dimensions are 1
  bool trainable;
  bool reg;        // in the L2 regulariser (regularized(name) of a trainable tensor)
};
// appends a tensor at n_params and advances n_params, keeping every tensor 16-byte aligned inside the flat buffer; returns its offset
long long add_param(std::vector<Param>& table, long long& n_params, const std::string& name, std::initializer_list<int> shape,
                    bool trainable = true);
bool regularized(const std::string& name);
// offsets of a convolution + batch-norm block's tensors
struct ConvBnParams { long long kernel, bias, gamma, beta, mm, mv; };
// prefix + kernel [k][cin][cout], bias, gamma, beta (trainable) and moving_mean, moving_variance [cout], in that order
ConvBnParams add_conv_bn_params(std::vector<Param>& table, long long& n_params, const std::string& prefix, int k, int cin, int cout);
// the out-parameters of the *_param_info C-ABI functions; offset, ndim, shape4 and trainable may be NULL
int param_info(const std::vector<Param>& table, int i, char* name, int cap, long long* offset, int* ndim, int* shape4, int* trainable);

// fp32 [K][N] (TensorFlow [in][out]) -> bf16 GEMM operand: transpose: dst[row(n)][col0 + k], else dst[k][col0 + n]
struct PackJob {
  long long src_off;  // fp32 element offset in params
  int K, N;
  long long dst_off;  // bf16 element offset in packed
  int dst_ld;
  int transpose;
  int col0;
  float scale;
  int perm;           // > 0 (transposing jobs): column n = g * perm + u is a gate-major column; see launch_pack for its row
  int part;           // 0 / 1: bf16(w) ; 2: bf16(w - bf16(w)), the low half of the split-bf16 operand
};
void add_pack(std::vector<PackJob>& jobs, long long src, int K, int N, long long dst_bytes, int ld, int transpose, int col0, float scale = 1.f,
              int perm = 0);
// Forward GEMM operands: packed bf16 weights [rows][Kw], K contiguous, whose columns the GEMM reads as plain segments of nkb 64-wide
// blocks over nlayers layer slabs (Seg, t2_gemm_types.h). In the split-bf16 ("fp32-class") mode the operand is [rows][3 Kw]: a plain
// segment that starts at column c and is Ks = nkb * 64 * nlayers wide has weight slots of Cp = nkb * 64 columns, and the slot at plain
// column c + x is packed at split columns 3c + 2x and 3c + 2x + Cp (W_hi, both read against activation rows [hi | lo]) and 3c + 2Ks + x
// (W_lo, read against the hi half). With one layer that is [W_hi | W_hi | W_lo] per slot; over layers, every layer's [W_hi | W_hi] and
// then every layer's W_lo. The GEMM side of the rule is ActGemmCall::split (t2_gemm.h).
inline long long fwd_operand_bytes(long long rows, long long Kw, bool split) { return 2 * rows * Kw * (split ? 3 : 1); }
// fp32 [K][N] -> rows [0, N) of the forward operand at dst_bytes: the weight slot of `layer` in the plain segment that starts at column
// c and loops over `layers` slots of Cp columns
void add_pack_fwd(std::vector<PackJob>& jobs, bool split, long long src, int K, int N, long long dst_bytes, int Kw, int c, int Cp,
                  float scale = 1.f, int perm = 0, int layer = 0, int layers = 1);
// runs the jobs_dev[0, n_jobs) table at grid (grid_x, n_jobs) x (32, 8). W is the row block width of the gate permutation:
// row = (u / W) * (gates * W) + g * W + u % W, with W = 128 for WaveNet's two gate halves (tanh | sigmoid) and W = 32 for the four
// LSTM gates of the EPI_LSTM rows. The permutation is a bijection of the job's N rows only when the job transposes, N == gates * perm
// and perm % W == 0; the kernel does not check this, and a job that breaks it writes rows outside its block, so every job with
// perm > 0 must be built to meet it.
int launch_pack(const float* params, void* packed, const PackJob* jobs_dev, int n_jobs, int W, int grid_x, cudaStream_t st);

// L2 regulariser: the table holds (offset, elements) of every tensor with reg set; reg_loss adds 0.5 sum w^2 to *dst,
// reg_grad adds weight * w to the gradients
int upload_reg_table(const std::vector<Param>& table, void* dst, cudaStream_t st);
void launch_reg_loss(const float* params, const long long* tab, int n_reg, float* dst, cudaStream_t st);
void launch_reg_grad(const float* params, float* grads, const long long* tab, int n_reg, float weight, cudaStream_t st);

void launch_f32_to_bf16(const float* in, __nv_bfloat16* out, long long n, cudaStream_t st);
// fp32 [rows][C] -> split-bf16 operand rows [hi(Cp) | lo(Cp)] (row pitch 2 Cp, Cp >= C; the padding channels are written as zeros)
void launch_f32_to_bf16_split(const float* in, __nv_bfloat16* out, long long rows, int C, int Cp, cudaStream_t st);

// side stream with fork / join events for work that is independent of the caller's stream (created once per process;
// T2_SIDE_STREAM=0 in the environment keeps everything on the caller's stream: nullptr)
struct SideStream { cudaStream_t s; cudaEvent_t fork, fork2, join; };
SideStream* side_stream();

}  // namespace t2
