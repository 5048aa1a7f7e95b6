// t2_audio.cu — audio front-end kernels: fused STFT -> power -> mel -> dB -> normalise, pre-emphasis, mu-law.
//
// Replaces datasets/audio.py:22-25 (preemphasis), :61-77 (linearspectrogram / melspectrogram), :178-182 (_stft via
// librosa.stft, center=True, pad_mode='constant'), :225-270 (_linear_to_mel, _amp_to_db, _normalize) and
// wavenet_vocoder/util.py:30-129 (mu-law family) of the reference.
//
// Each frame is transformed by its own n_fft/32 threads of a 256-thread CTA: the Hann-windowed frame (only win_size of the
// n_fft samples are non-zero) is packed as n_fft/2 complex points, run through a register-radix Stockham FFT, untangled into
// the n_fft/2+1 real-FFT bins, raised to magnitude_power, contracted with the SPARSE triangular mel filters, converted to dB
// and normalised — one HBM read of the samples, one HBM write of num_mels floats per frame, nothing in between.
// The FFT runs in fp64: the reference's spectra come from a double-precision FFT (numpy) and the dB floor sits
// ~100 dB under the spectral peak, which fp32 butterflies cannot resolve to the 1e-3 parity tolerance.
// n_fft is 512, 1024, 2048 or 4096 (the reference's advice, hparams.py:52: the first power of two above win_size,
// i.e. 8, 16, 22.05-24 and 44.1-48 kHz audio); the FFT kernels are instantiated once per complex length N = n_fft / 2.
#include <math.h>
#include <string.h>

#include <cmath>
#include <type_traits>
#include <vector>

#include "../../include/t2b200.h"
#include "t2_common.cuh"

namespace t2 {
namespace {

constexpr int kMaxMels = 128;

bool nfft_supported(int n_fft) { return n_fft == 512 || n_fft == 1024 || n_fft == 2048 || n_fft == 4096; }
bool in_range(long long v, long long lo, long long hi) { return v >= lo && v <= hi; }

// calls f(std::integral_constant<int, N>) for the complex FFT length N = n_fft / 2 of a supported n_fft
template <class F>
int by_nfft(int n_fft, F&& f) {
  switch (n_fft) {
    case 512: return f(std::integral_constant<int, 256>());
    case 1024: return f(std::integral_constant<int, 512>());
    case 2048: return f(std::integral_constant<int, 1024>());
    case 4096: return f(std::integral_constant<int, 2048>());
    default: return t2_set_error(T2_ERR_UNSUPPORTED_SHAPE, "no audio kernel for n_fft %d", n_fft);
  }
}

struct Plan {
  // byte offsets inside the device plan buffer
  long long o_tw, o_tw2, o_win, o_fstart, o_fcount, o_foff, o_fw;
  long long bytes;
  int nnz;
};

inline long long al(long long v) { return (v + 255) / 256 * 256; }

double hz_to_mel(double f) {
  const double f_sp = 200.0 / 3, min_log_hz = 1000.0, min_log_mel = min_log_hz / f_sp, logstep = log(6.4) / 27.0;
  return f >= min_log_hz ? min_log_mel + log(f / min_log_hz) / logstep : f / f_sp;
}
double mel_to_hz(double m) {
  const double f_sp = 200.0 / 3, min_log_hz = 1000.0, min_log_mel = min_log_hz / f_sp, logstep = log(6.4) / 27.0;
  return m >= min_log_mel ? min_log_hz * exp(logstep * (m - min_log_mel)) : f_sp * m;
}

// librosa.filters.mel (Slaney scale, area normalised), dense [n_mels][bins] in double
void mel_basis(const t2_audio_config_t& c, std::vector<double>& W) {
  const int nm = c.num_mels, bins = c.n_fft / 2 + 1;
  W.assign(size_t(nm) * bins, 0.0);
  std::vector<double> mel_f(nm + 2);
  const double m0 = hz_to_mel(c.fmin), m1 = hz_to_mel(c.fmax);
  for (int i = 0; i < nm + 2; ++i) mel_f[i] = mel_to_hz(m0 + (m1 - m0) * i / (nm + 1));
  for (int i = 0; i < nm; ++i) {
    const double enorm = 2.0 / (mel_f[i + 2] - mel_f[i]);
    for (int k = 0; k < bins; ++k) {
      const double f = double(c.sample_rate) / 2 * k / (bins - 1);
      const double lower = (f - mel_f[i]) / (mel_f[i + 1] - mel_f[i]);
      const double upper = (mel_f[i + 2] - f) / (mel_f[i + 2] - mel_f[i + 1]);
      const double w = fmax(0.0, fmin(lower, upper));
      W[size_t(i) * bins + k] = w * enorm;
    }
  }
}

int make_plan(const t2_audio_config_t* c, Plan& p, std::vector<double>* basis_out) {
  T2_REQUIRE(c != nullptr, T2_ERR_INVALID_ARG, "null audio config");
  T2_REQUIRE(nfft_supported(c->n_fft), T2_ERR_UNSUPPORTED_SHAPE,
             "n_fft must be 512, 1024, 2048 or 4096 (got %d): the first power of two above win_size (hparams.py:52)", c->n_fft);
  T2_REQUIRE(c->win_size >= 2 && c->win_size <= c->n_fft && c->hop_size >= 1, T2_ERR_INVALID_ARG, "bad win/hop");
  T2_REQUIRE(c->num_mels >= 1 && c->num_mels <= kMaxMels, T2_ERR_UNSUPPORTED_SHAPE, "num_mels out of range");
  T2_REQUIRE(c->fmax <= c->sample_rate / 2 && c->fmin >= 0, T2_ERR_INVALID_ARG, "bad fmin/fmax");
  std::vector<double> W;
  mel_basis(*c, W);
  int nnz = 0;
  for (double w : W) nnz += w != 0.0;
  const int N = c->n_fft / 2;
  long long o = 0;
  p.o_tw = o; o = al(o + N * 16);
  p.o_tw2 = o; o = al(o + (N / 2 + 1) * 16);
  p.o_win = o; o = al(o + c->win_size * 8);
  p.o_fstart = o; o = al(o + c->num_mels * 4);
  p.o_fcount = o; o = al(o + c->num_mels * 4);
  p.o_foff = o; o = al(o + c->num_mels * 4);
  p.o_fw = o; o = al(o + (long long)(nnz + 1) * 8);
  p.bytes = o;
  p.nnz = nnz;
  if (basis_out) basis_out->swap(W);
  return T2_OK;
}

struct StftArgs {
  const float* wav;       // [B][n_samples]
  float* mel;             // [B][frames][nm] or [B][nm][frames]
  float* lin;             // nullable, [B][frames][bins] or [B][bins][frames]
  const double2* tw;      // W_N^k, k = 0..N-1 (N = n_fft / 2)
  const double2* tw2;     // W_n_fft^k, k = 0..N/2
  const double* win;      // periodic Hann, win_size
  const int* fstart; const int* fcount; const int* foff; const double* fw;
  int B, n_samples, frames, hop, win_size, nm, time_major;
  float preemph, gain, mag_power;
  float min_level, min_level_db, ref_level_db, max_abs;
  int normalize, symmetric, clip;
};

__device__ __forceinline__ double2 cmul(double2 a, double2 b) {
  return make_double2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}

__device__ __forceinline__ float finish(const StftArgs& a, double v) {
  // _amp_to_db (audio.py:248-250) - ref_level_db, then _normalize (audio.py:258-270)
  float s = 20.f * log10f(fmaxf(a.min_level, float(v))) - a.ref_level_db;
  if (!a.normalize) return s;
  float r;
  if (a.symmetric) r = (2.f * a.max_abs) * ((s - a.min_level_db) / (-a.min_level_db)) - a.max_abs;
  else r = a.max_abs * ((s - a.min_level_db) / (-a.min_level_db));
  if (a.clip) r = fminf(fmaxf(r, a.symmetric ? -a.max_abs : 0.f), a.max_abs);
  return r;
}

// ---- register-radix FFT, 4096 / N frames per CTA ----------------------------------------------------------------------------
// N / 16 threads own one frame (16 complex points each); N = 16 x 16 x R Stockham passes (R = N / 256 = 1, 2, 4 or 8) with the
// radix-16 butterflies held in registers, so a frame crosses shared memory at most three times and never needs a CTA-wide
// barrier: the threads of a frame meet on their own named barrier, or on a half-warp __syncwarp when a frame is 16 threads. The
// first pass reads the windowed samples straight from global memory (no staging pass). Shared-memory rows are padded by one
// element per 16 (17 j + r) so that the transposing stores of the radix-16 passes are conflict-free for 16-byte elements. The
// CTA is 256 threads for every N and a frame's shared memory grows with N, so every size keeps ~102.5 KB per CTA and 2 CTAs per SM.
constexpr int kCtaThreads = 256;
template <int N>
struct FftShape {
  static_assert(N == 256 || N == 512 || N == 1024 || N == 2048, "complex FFT length N = n_fft / 2");
  static constexpr int kFrameThreads = N / 16;
  static constexpr int kFramesPerCta = kCtaThreads / kFrameThreads;
  static constexpr int kPadN = N + N / 16;                    // padded complex buffer
  static constexpr int kPwN = N + 8;                          // N + 1 power-spectrum bins, padded
  static constexpr int kSmemBytes = kFramesPerCta * (kPadN * 16 + kPwN * 8);
};
static_assert(FftShape<1024>::kSmemBytes == 102656, "n_fft = 2048 keeps its shared-memory footprint");

__device__ __forceinline__ int padi(int i) { return i + (i >> 4); }
// the T threads of frame `slot` meet; T >= 32: named barrier slot + 1 (at most 8 frames per CTA), T = 16: half a warp
template <int T>
__device__ __forceinline__ void frame_sync(int slot) {
  if constexpr (T >= 32) asm volatile("bar.sync %0, %1;" ::"r"(slot + 1), "n"(T) : "memory");
  else __syncwarp(((1u << T) - 1) << (T * (slot & (32 / T - 1))));
}
__device__ __forceinline__ double2 cadd(double2 a, double2 b) { return make_double2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ double2 csub(double2 a, double2 b) { return make_double2(a.x - b.x, a.y - b.y); }
// forward DFT-4 in place: (a, b, c, d) -> (X0, X1, X2, X3)
__device__ __forceinline__ void dft4(double2& a, double2& b, double2& c, double2& d) {
  const double2 s02 = cadd(a, c), d02 = csub(a, c), s13 = cadd(b, d), d13 = csub(b, d);
  a = cadd(s02, s13);
  b = make_double2(d02.x + d13.y, d02.y - d13.x);   // d02 - i d13
  c = csub(s02, s13);
  d = make_double2(d02.x - d13.y, d02.y + d13.x);   // d02 + i d13
}
// forward DFT-16 of v[0..15] (natural order in, natural order out) as 4 x 4 with the W16 twiddles as constants
__device__ __forceinline__ void dft16(double2* v) {
  constexpr double c1 = 0.92387953251128675613, s1 = 0.38268343236508977173, h = 0.70710678118654752440;
#pragma unroll
  for (int n2 = 0; n2 < 4; ++n2) dft4(v[n2], v[4 + n2], v[8 + n2], v[12 + n2]);   // v[4 k1 + n2] = y[n2][k1]
  // y[n2][k1] *= W16^(n2 k1)
  v[4 + 1] = cmul(v[4 + 1], make_double2(c1, -s1));     // n2=1,k1=1: W^1
  v[8 + 1] = cmul(v[8 + 1], make_double2(h, -h));       // n2=1,k1=2: W^2
  v[12 + 1] = cmul(v[12 + 1], make_double2(s1, -c1));   // n2=1,k1=3: W^3
  v[4 + 2] = cmul(v[4 + 2], make_double2(h, -h));       // n2=2,k1=1: W^2
  v[8 + 2] = make_double2(v[8 + 2].y, -v[8 + 2].x);     // n2=2,k1=2: W^4 = -i
  v[12 + 2] = cmul(v[12 + 2], make_double2(-h, -h));    // n2=2,k1=3: W^6
  v[4 + 3] = cmul(v[4 + 3], make_double2(s1, -c1));     // n2=3,k1=1: W^3
  v[8 + 3] = cmul(v[8 + 3], make_double2(-h, -h));      // n2=3,k1=2: W^6
  v[12 + 3] = cmul(v[12 + 3], make_double2(-c1, s1));   // n2=3,k1=3: W^9
#pragma unroll
  for (int k1 = 0; k1 < 4; ++k1) dft4(v[4 * k1], v[4 * k1 + 1], v[4 * k1 + 2], v[4 * k1 + 3]);  // -> X[k1 + 4 k2] at v[4 k1 + k2]
  // transpose the 4 x 4 register tile so that v[k] = X[k]
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = i + 1; j < 4; ++j) { const double2 t = v[4 * i + j]; v[4 * i + j] = v[4 * j + i]; v[4 * j + i] = t; }
}

// forward DFT-8 of v[0..7] (natural order in and out) as 2 x 4: X[k] = E[k] + W8^k O[k], X[k + 4] = E[k] - W8^k O[k]
__device__ __forceinline__ void dft8(double2* v) {
  constexpr double h = 0.70710678118654752440;
  dft4(v[0], v[2], v[4], v[6]);                                   // E[k] at v[2 k]
  dft4(v[1], v[3], v[5], v[7]);                                   // O[k] at v[2 k + 1]
  const double2 o[4] = {v[1], cmul(v[3], make_double2(h, -h)), make_double2(v[5].y, -v[5].x), cmul(v[7], make_double2(-h, -h))};
  const double2 e[4] = {v[0], v[2], v[4], v[6]};
#pragma unroll
  for (int k = 0; k < 4; ++k) { v[k] = cadd(e[k], o[k]); v[k + 4] = csub(e[k], o[k]); }
}
// forward DFT-R of v[0..R-1] in place, natural order in and out
template <int R>
__device__ __forceinline__ void dft_small(double2* v) {
  if constexpr (R == 2) { const double2 t = v[1]; v[1] = csub(v[0], t); v[0] = cadd(v[0], t); }
  else if constexpr (R == 4) dft4(v[0], v[1], v[2], v[3]);
  else dft8(v);
}

// The Stockham passes of the N-point forward FFT of one frame (T = N / 16 threads). In: v[r] = z[j + T r] (thread j of the
// frame's T). Out: the transform in natural order in `buf` (padded index padi(k)), visible to all T threads of the frame.
template <int N>
__device__ __forceinline__ void fft_passes(double2 (&v)[16], double2* buf, const double2* __restrict__ tw, int slot, int j) {
    constexpr int T = N / 16, R = N / 256;
    dft16(v);
#pragma unroll
    for (int r = 0; r < 16; ++r) buf[17 * j + r] = v[r];          // padi(16 j + r)
    frame_sync<T>(slot);
    // pass 2 (radix 16, Ns = 16): twiddle W_256^(r k) = W_N^(R r k)
    {
      const int k = j & 15;
#pragma unroll
      for (int r = 0; r < 16; ++r) v[r] = buf[padi(j + T * r)];
#pragma unroll
      for (int r = 1; r < 16; ++r) v[r] = cmul(v[r], __ldg(tw + R * r * k));
      dft16(v);
      frame_sync<T>(slot);
      const int base = (j - k) * 16 + k;
#pragma unroll
      for (int r = 0; r < 16; ++r) buf[padi(base + 16 * r)] = v[r];
    }
    frame_sync<T>(slot);
    if constexpr (R > 1) {
      // pass 3 (radix R, Ns = 256): 16 / R butterflies per thread, output in natural order
#pragma unroll
      for (int u = 0; u < 16 / R; ++u) {
        const int jj = j + T * u;
        v[R * u] = buf[padi(jj)];
#pragma unroll
        for (int r = 1; r < R; ++r) v[R * u + r] = cmul(buf[padi(jj + 256 * r)], __ldg(tw + r * jj));
        dft_small<R>(v + R * u);
      }
      frame_sync<T>(slot);
#pragma unroll
      for (int u = 0; u < 16 / R; ++u)
#pragma unroll
        for (int r = 0; r < R; ++r) buf[padi(j + T * u + 256 * r)] = v[R * u + r];
      frame_sync<T>(slot);
    }
}

template <int N>
__global__ void __launch_bounds__(kCtaThreads, 2) stft_mel_kernel_v2(StftArgs a) {
  using S = FftShape<N>;
  constexpr int T = S::kFrameThreads, F = S::kFramesPerCta;
  extern __shared__ __align__(16) uint8_t smem_v2[];
  const int slot = threadIdx.x / T;
  const int j = threadIdx.x % T;
  double2* buf = reinterpret_cast<double2*>(smem_v2) + slot * S::kPadN;
  double* pw = reinterpret_cast<double*>(smem_v2 + F * S::kPadN * 16) + slot * S::kPwN;
  const long long total = (long long)a.B * a.frames;
  const int lpad = (2 * N - a.win_size) / 2;
  for (long long fr = (long long)blockIdx.x * F + slot; fr < total; fr += (long long)gridDim.x * F) {
    const int b = int(fr / a.frames), f = int(fr % a.frames);
    const float* w = a.wav + (long long)b * a.n_samples;
    double2 v[16];
    // pass 1 (radix 16, Ns = 1): v[r] = z[j + T r], z[n] = x[2n] + i x[2n+1] (windowed, centred, zero padded)
#pragma unroll
    for (int r = 0; r < 16; ++r) {
      const int q0 = 2 * (j + T * r);
      double c[2];
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int q = q0 + hh, wi = q - lpad;
        double s = 0.0;
        if (wi >= 0 && wi < a.win_size) {
          const long long si = (long long)f * a.hop - N + q;
          if (si >= 0 && si < a.n_samples) {
            double x = double(__ldg(w + si));
            if (a.preemph != 0.f) x -= double(a.preemph) * (si > 0 ? double(__ldg(w + si - 1)) : 0.0);
            s = x * double(a.gain) * __ldg(a.win + wi);
          }
        }
        c[hh] = s;
      }
      v[r] = make_double2(c[0], c[1]);
    }
    fft_passes<N>(v, buf, a.tw, slot, j);
    // untangle to the real-FFT bins and take |X|^p; librosa stores the STFT as complex64 before |.|: round the components like the
    // reference does, then np.abs(complex64) -> float32 and ** p in float32
    for (int k = j; k <= N; k += T) {
      const double2 zk = buf[padi(k & (N - 1))];
      const double2 zn = buf[padi((N - k) & (N - 1))];
      const double2 e = make_double2(0.5 * (zk.x + zn.x), 0.5 * (zk.y - zn.y));
      const double2 o = make_double2(0.5 * (zk.y + zn.y), -0.5 * (zk.x - zn.x));
      const int kk = k <= N / 2 ? k : N - k;
      double2 t2w = __ldg(a.tw2 + kk);
      if (k > N / 2) t2w = make_double2(-t2w.x, t2w.y);
      const double2 ow = cmul(o, t2w);
      const float ref = float(e.x + ow.x), imf = float(e.y + ow.y);
      const double mag2 = double(ref) * double(ref) + double(imf) * double(imf);
      double val;
      if (a.mag_power == 2.f) {
        const float m = sqrtf(float(mag2));
        val = double(m * m);
      } else {
        val = double(powf(sqrtf(float(mag2)), a.mag_power));
      }
      pw[k] = val;
      if (a.lin) {
        const float r = finish(a, val);
        if (a.time_major) a.lin[((long long)b * a.frames + f) * (N + 1) + k] = r;
        else a.lin[((long long)b * (N + 1) + k) * a.frames + f] = r;
      }
    }
    frame_sync<T>(slot);
    // sparse mel filterbank: one thread per filter (the long high-frequency filters pair up with the short low ones)
    for (int m = j; m < a.nm; m += T) {
      const int s = __ldg(a.fstart + m), n = __ldg(a.fcount + m);
      const double* fw = a.fw + __ldg(a.foff + m);
      double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0;   // four independent chains: the longest filter spans ~70 bins at n_fft = 2048
      int i = 0;
      for (; i + 4 <= n; i += 4) {
        a0 += __ldg(fw + i) * pw[s + i];
        a1 += __ldg(fw + i + 1) * pw[s + i + 1];
        a2 += __ldg(fw + i + 2) * pw[s + i + 2];
        a3 += __ldg(fw + i + 3) * pw[s + i + 3];
      }
      for (; i < n; ++i) a0 += __ldg(fw + i) * pw[s + i];
      const double acc = (a0 + a1) + (a2 + a3);
      const float r = finish(a, acc);
      if (a.time_major) a.mel[((long long)b * a.frames + f) * a.nm + m] = r;
      else a.mel[((long long)b * a.nm + m) * a.frames + f] = r;
    }
    frame_sync<T>(slot);
  }
}

// ---- Griffin-Lim (datasets/audio.py:151-161 _griffin_lim, :184-186 _istft = librosa.istft, :178-182 _stft) ------------------------
// One iteration = three kernels over [B][frames]:
//   gl_istft_kernel   per frame: X = S * phase -> inverse real FFT (the forward machinery on conj(Z), Z the packed half-length
//                     spectrum) -> multiply by the synthesis window -> the win_size non-zero samples of the frame
//   gl_ola_kernel     overlap-add of the <= ceil(win / hop) frames covering a sample, divided by the window sum of squares
//                     (librosa.istft), centre trim of n_fft / 2
//   gl_stft_kernel    STFT of the new signal -> unit phases exp(i angle(X)) for the next iteration
struct GlArgs {
  const float* mag;       // [B][frames][bins] magnitudes S
  float2* phase;          // [B][frames][bins] unit phases
  float* fr;              // [B][frames][win] windowed time-domain frames
  float* y;               // [B][n_out]
  const double2* tw; const double2* tw2; const double* win;
  int B, frames, hop, win_size, n_out, n_fft;
};
template <int N>
__global__ void __launch_bounds__(kCtaThreads, 2) gl_istft_kernel(GlArgs a) {
  using Sh = FftShape<N>;
  constexpr int T = Sh::kFrameThreads, F = Sh::kFramesPerCta;
  extern __shared__ __align__(16) uint8_t smem_v2[];
  const int slot = threadIdx.x / T, j = threadIdx.x % T;
  double2* buf = reinterpret_cast<double2*>(smem_v2) + slot * Sh::kPadN;
  const long long total = (long long)a.B * a.frames;
  const int lpad = (2 * N - a.win_size) / 2;
  for (long long fr = (long long)blockIdx.x * F + slot; fr < total; fr += (long long)gridDim.x * F) {
    const float* S = a.mag + fr * (N + 1);
    const float2* ph = a.phase + fr * (N + 1);
    double2 v[16];
#pragma unroll
    for (int r = 0; r < 16; ++r) {
      const int k = j + T * r;                      // Z[k] = E[k] + i O[k], E / O from X[k] and conj(X[N - k])
      const float sk = S[k], sn = S[N - k];
      const float2 pk = ph[k], pn = ph[N - k];
      double2 xk = make_double2(double(sk) * pk.x, double(sk) * pk.y);
      double2 xn = make_double2(double(sn) * pn.x, -double(sn) * pn.y);           // conj(X[N - k])
      if (k == 0) { xk.y = 0.0; xn.y = 0.0; }       // a real inverse transform ignores the imaginary parts of the DC / Nyquist bins (np.fft.irfft)
      const double2 e = make_double2(0.5 * (xk.x + xn.x), 0.5 * (xk.y + xn.y));
      const double2 d = make_double2(0.5 * (xk.x - xn.x), 0.5 * (xk.y - xn.y));
      const int kk = k <= N / 2 ? k : N - k;
      double2 w = __ldg(a.tw2 + kk);                // W_n_fft^kk = exp(-2 pi i kk / n_fft); needed: exp(+2 pi i k / n_fft)
      w = k <= N / 2 ? make_double2(w.x, -w.y) : make_double2(-w.x, -w.y);         // k > n_fft/4: exp(+i pi (N - kk) / N) = -conj(exp(+..kk))
      const double2 o = cmul(d, w);
      const double2 z = make_double2(e.x - o.y, e.y + o.x);                       // E + i O
      v[r] = make_double2(z.x, -z.y);               // conj: the inverse transform is conj(FFT(conj(Z))) / N
    }
    fft_passes<N>(v, buf, a.tw, slot, j);
    float* out = a.fr + fr * a.win_size;
    for (int wi = j; wi < a.win_size; wi += T) {
      const int q = wi + lpad;                      // sample q of the n_fft frame = (q even ? Re : Im) z[q / 2], z = conj(W) / N
      const double2 wv = buf[padi(q >> 1)];
      const double x = ((q & 1) ? -wv.y : wv.x) * (1.0 / N);
      out[wi] = float(x * __ldg(a.win + wi));
    }
    frame_sync<T>(slot);
  }
}
__global__ void gl_ola_kernel(GlArgs a) {
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e >= (long long)a.B * a.n_out) return;
  const int b = int(e / a.n_out), n = int(e % a.n_out);
  const int lpad = (a.n_fft - a.win_size) / 2;
  const int p = n + a.n_fft / 2 - lpad;             // position relative to the window support of frame 0
  int k1 = p / a.hop;
  if (k1 > a.frames - 1) k1 = a.frames - 1;
  float acc = 0.f, wss = 0.f;
  for (int k = k1; k >= 0; --k) {
    const int wi = p - k * a.hop;
    if (wi >= a.win_size) break;
    const float w = float(__ldg(a.win + wi));
    acc += a.fr[((long long)b * a.frames + k) * a.win_size + wi];
    wss += w * w;
  }
  a.y[e] = wss > 1.17549435e-38f ? acc / wss : acc;
}
template <int N>
__global__ void __launch_bounds__(kCtaThreads, 2) gl_stft_kernel(GlArgs a) {
  using Sh = FftShape<N>;
  constexpr int T = Sh::kFrameThreads, F = Sh::kFramesPerCta;
  extern __shared__ __align__(16) uint8_t smem_v2[];
  const int slot = threadIdx.x / T, j = threadIdx.x % T;
  double2* buf = reinterpret_cast<double2*>(smem_v2) + slot * Sh::kPadN;
  const long long total = (long long)a.B * a.frames;
  const int lpad = (2 * N - a.win_size) / 2;
  for (long long fr = (long long)blockIdx.x * F + slot; fr < total; fr += (long long)gridDim.x * F) {
    const int b = int(fr / a.frames), f = int(fr % a.frames);
    const float* w = a.y + (long long)b * a.n_out;
    double2 v[16];
#pragma unroll
    for (int r = 0; r < 16; ++r) {
      const int q0 = 2 * (j + T * r);
      double c[2];
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int q = q0 + hh, wi = q - lpad;
        double sv = 0.0;
        if (wi >= 0 && wi < a.win_size) {
          const long long si = (long long)f * a.hop - N + q;
          if (si >= 0 && si < a.n_out) sv = double(__ldg(w + si)) * __ldg(a.win + wi);
        }
        c[hh] = sv;
      }
      v[r] = make_double2(c[0], c[1]);
    }
    fft_passes<N>(v, buf, a.tw, slot, j);
    float2* ph = a.phase + fr * (N + 1);
    for (int k = j; k <= N; k += T) {
      const double2 zk = buf[padi(k & (N - 1))];
      const double2 zn = buf[padi((N - k) & (N - 1))];
      const double2 e = make_double2(0.5 * (zk.x + zn.x), 0.5 * (zk.y - zn.y));
      const double2 o = make_double2(0.5 * (zk.y + zn.y), -0.5 * (zk.x - zn.x));
      const int kk = k <= N / 2 ? k : N - k;
      double2 t2w = __ldg(a.tw2 + kk);
      if (k > N / 2) t2w = make_double2(-t2w.x, t2w.y);
      const double2 ow = cmul(o, t2w);
      const float re = float(e.x + ow.x), im = float(e.y + ow.y);   // complex64 like librosa's STFT matrix
      const float m = sqrtf(re * re + im * im);
      ph[k] = m > 0.f ? make_float2(re / m, im / m) : make_float2(1.f, 0.f);      // np.angle(0) = 0
    }
    frame_sync<T>(slot);
  }
}
// initial phases exp(2 pi i u), u from the counter hash (the reference draws np.random.rand)
__global__ void gl_init_phase_kernel(float2* __restrict__ ph, long long n, unsigned long long seed) {
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e >= n) return;
  float sn, cs;
  sincospif(2.f * hash_uniform(seed, (unsigned long long)e), &sn, &cs);
  ph[e] = make_float2(cs, sn);
}

__global__ void preemphasis_kernel(const float* __restrict__ x, float* __restrict__ y, long long n_per, long long n, float k) {
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e >= n) return;
  const long long i = e % n_per;
  y[e] = float(double(x[e]) - double(k) * (i > 0 ? double(x[e - 1]) : 0.0));
}

// mu-law, float32 pipeline of wavenet_vocoder/util.py:30-102 (see oracle/audio.py for the dtype definition):
// log1p is evaluated in fp64 and rounded to fp32 (a correctly-rounded log1pf); every other step is an IEEE fp32 op.
__device__ __forceinline__ float mulaw_f(float x) {
  const float a = __fmul_rn(255.0f, fabsf(x));
  const float l = float(log1p(double(a)));
  const float den = float(log1p(255.0));
  const float sg = x > 0.f ? 1.f : (x < 0.f ? -1.f : 0.f);
  return __fdiv_rn(__fmul_rn(sg, l), den);
}
__global__ void mulaw_quantize_kernel(const float* __restrict__ x, int* __restrict__ q, long long n) {
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e >= n) return;
  const float y = mulaw_f(x[e]);
  const float s = __fmul_rn(__fdiv_rn(__fadd_rn(y, 1.0f), 2.0f), 255.0f);
  q[e] = int(s);  // truncation toward zero == astype(np.int) / tf.cast(int32)
}
__global__ void mulaw_kernel(const float* __restrict__ x, float* __restrict__ y, long long n) {
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e < n) y[e] = mulaw_f(x[e]);
}
__device__ __forceinline__ float inv_mulaw_f(float y) {
  const float p = float(pow(256.0, double(fabsf(y))));
  const float sg = y > 0.f ? 1.f : (y < 0.f ? -1.f : 0.f);
  return __fmul_rn(__fmul_rn(sg, float(1.0 / 255.0)), __fadd_rn(p, -1.0f));
}
__global__ void inv_mulaw_kernel(const float* __restrict__ y, float* __restrict__ x, long long n) {
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e < n) x[e] = inv_mulaw_f(y[e]);
}
__global__ void inv_mulaw_quantize_kernel(const int* __restrict__ q, float* __restrict__ x, long long n) {
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e >= n) return;
  const float y = __fadd_rn(__fdiv_rn(__fmul_rn(2.0f, float(q[e])), 255.0f), -1.0f);
  x[e] = inv_mulaw_f(y);
}

inline unsigned nblk(long long n) { return (unsigned)((n + 255) / 256); }

// grid of the frame-parallel kernels: 2 resident CTAs per SM (~102.5 KB smem, 256 threads, <= 128 registers each)
template <int N>
unsigned frame_grid(long long frames, int sms) {
  const long long groups = (frames + FftShape<N>::kFramesPerCta - 1) / FftShape<N>::kFramesPerCta, cap = (long long)sms * 2;
  return (unsigned)(groups < cap ? groups : cap);
}

template <int N>
int launch_stft_mel(const StftArgs& a, int sms, cudaStream_t st) {
  constexpr int smem = FftShape<N>::kSmemBytes;
  static bool configured = false;
  if (!configured) {
    T2_CHECK_CUDA(cudaFuncSetAttribute(stft_mel_kernel_v2<N>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    configured = true;
  }
  stft_mel_kernel_v2<N><<<frame_grid<N>((long long)a.B * a.frames, sms), kCtaThreads, smem, st>>>(a); t2_count_launch();
  return T2_OK;
}

// One launcher per Griffin-Lim kernel, shared by launch_griffin_lim and t2_dbg_audio_kernel.
template <int N>
int launch_gl_istft(const GlArgs& a, int sms, cudaStream_t st) {
  constexpr int smem = FftShape<N>::kSmemBytes;
  static bool configured = false;
  if (!configured) {
    T2_CHECK_CUDA(cudaFuncSetAttribute(gl_istft_kernel<N>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    configured = true;
  }
  gl_istft_kernel<N><<<frame_grid<N>((long long)a.B * a.frames, sms), kCtaThreads, smem, st>>>(a); t2_count_launch();
  return T2_OK;
}
template <int N>
int launch_gl_stft(const GlArgs& a, int sms, cudaStream_t st) {
  constexpr int smem = FftShape<N>::kSmemBytes;
  static bool configured = false;
  if (!configured) {
    T2_CHECK_CUDA(cudaFuncSetAttribute(gl_stft_kernel<N>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    configured = true;
  }
  gl_stft_kernel<N><<<frame_grid<N>((long long)a.B * a.frames, sms), kCtaThreads, smem, st>>>(a); t2_count_launch();
  return T2_OK;
}
void launch_gl_ola(const GlArgs& a, cudaStream_t st) {
  const long long ny = (long long)a.B * a.n_out;
  gl_ola_kernel<<<nblk(ny), 256, 0, st>>>(a); t2_count_launch();
}
void launch_gl_init_phase(float2* ph, long long n, unsigned long long seed, cudaStream_t st) {
  gl_init_phase_kernel<<<nblk(n), 256, 0, st>>>(ph, n, seed); t2_count_launch();
}

template <int N>
int launch_griffin_lim(const GlArgs& a, int iters, bool init_phase, unsigned long long seed, int sms, cudaStream_t st) {
  if (init_phase) launch_gl_init_phase(a.phase, (long long)a.B * a.frames * (N + 1), seed, st);
  for (int it = 0; it <= iters; ++it) {
    int rc = launch_gl_istft<N>(a, sms, st);
    if (rc) return rc;
    launch_gl_ola(a, st);
    if (it < iters && (rc = launch_gl_stft<N>(a, sms, st))) return rc;
  }
  return T2_OK;
}

int device_sms() {
  int dev = 0, sms = 148;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return sms;
}

// the kernel arguments of t2_stft_mel_f32 / t2_griffin_lim_f32 for a checked config, its plan and the caller's buffers
StftArgs stft_args(const t2_audio_config_t* cfg, const Plan& p, const void* d_plan, const float* wav, int B, int n_samples,
                   float preemphasis, float gain, float* mel, float* lin, int time_major) {
  const uint8_t* pl = static_cast<const uint8_t*>(d_plan);
  StftArgs a;
  memset(&a, 0, sizeof(a));
  a.wav = wav; a.mel = mel; a.lin = lin;
  a.tw = reinterpret_cast<const double2*>(pl + p.o_tw);
  a.tw2 = reinterpret_cast<const double2*>(pl + p.o_tw2);
  a.win = reinterpret_cast<const double*>(pl + p.o_win);
  a.fstart = reinterpret_cast<const int*>(pl + p.o_fstart);
  a.fcount = reinterpret_cast<const int*>(pl + p.o_fcount);
  a.foff = reinterpret_cast<const int*>(pl + p.o_foff);
  a.fw = reinterpret_cast<const double*>(pl + p.o_fw);
  a.B = B; a.n_samples = n_samples; a.frames = 1 + n_samples / cfg->hop_size; a.hop = cfg->hop_size;
  a.win_size = cfg->win_size; a.nm = cfg->num_mels; a.time_major = time_major;
  a.preemph = preemphasis; a.gain = gain; a.mag_power = cfg->magnitude_power;
  a.min_level = float(exp(double(cfg->min_level_db) / 20.0 * log(10.0)));
  a.min_level_db = cfg->min_level_db; a.ref_level_db = cfg->ref_level_db; a.max_abs = cfg->max_abs_value;
  a.normalize = cfg->signal_normalization; a.symmetric = cfg->symmetric_mels; a.clip = cfg->allow_clipping_in_normalization;
  return a;
}
GlArgs gl_args(const t2_audio_config_t* cfg, const Plan& p, const void* d_plan, int B, int frames) {
  const uint8_t* pl = static_cast<const uint8_t*>(d_plan);
  GlArgs a;
  memset(&a, 0, sizeof(a));
  a.tw = reinterpret_cast<const double2*>(pl + p.o_tw);
  a.tw2 = reinterpret_cast<const double2*>(pl + p.o_tw2);
  a.win = reinterpret_cast<const double*>(pl + p.o_win);
  a.B = B; a.frames = frames; a.hop = cfg->hop_size; a.win_size = cfg->win_size; a.n_out = cfg->hop_size * (frames - 1);
  a.n_fft = cfg->n_fft;
  return a;
}

}  // namespace
}  // namespace t2

using namespace t2;

extern "C" int t2_stft_mel_plan_bytes(const t2_audio_config_t* cfg, long long* bytes) {
  Plan p;
  int rc = make_plan(cfg, p, nullptr);
  if (rc) return rc;
  *bytes = p.bytes;
  return T2_OK;
}

extern "C" int t2_stft_mel_plan_init(const t2_audio_config_t* cfg, void* d_plan, void* stream) {
  Plan p;
  std::vector<double> W;
  int rc = make_plan(cfg, p, &W);
  if (rc) return rc;
  std::vector<uint8_t> h(p.bytes, 0);
  const int n_fft = cfg->n_fft, N = n_fft / 2;
  double* tw = reinterpret_cast<double*>(h.data() + p.o_tw);
  for (int k = 0; k < N; ++k) { tw[2 * k] = cos(-2.0 * M_PI * k / N); tw[2 * k + 1] = sin(-2.0 * M_PI * k / N); }
  double* tw2 = reinterpret_cast<double*>(h.data() + p.o_tw2);
  for (int k = 0; k <= N / 2; ++k) { tw2[2 * k] = cos(-2.0 * M_PI * k / n_fft); tw2[2 * k + 1] = sin(-2.0 * M_PI * k / n_fft); }
  double* win = reinterpret_cast<double*>(h.data() + p.o_win);
  for (int n = 0; n < cfg->win_size; ++n) win[n] = 0.5 - 0.5 * cos(2.0 * M_PI * n / cfg->win_size);  // periodic Hann
  int* fstart = reinterpret_cast<int*>(h.data() + p.o_fstart);
  int* fcount = reinterpret_cast<int*>(h.data() + p.o_fcount);
  int* foff = reinterpret_cast<int*>(h.data() + p.o_foff);
  double* fw = reinterpret_cast<double*>(h.data() + p.o_fw);
  const int bins = cfg->n_fft / 2 + 1;
  int off = 0;
  for (int m = 0; m < cfg->num_mels; ++m) {
    int s = -1, e = -1;
    for (int k = 0; k < bins; ++k)
      if (W[size_t(m) * bins + k] != 0.0) { if (s < 0) s = k; e = k; }
    fstart[m] = s < 0 ? 0 : s;
    fcount[m] = s < 0 ? 0 : e - s + 1;
    foff[m] = off;
    for (int k = 0; k < fcount[m]; ++k) fw[off + k] = W[size_t(m) * bins + fstart[m] + k];
    off += fcount[m];
  }
  T2_REQUIRE(off <= p.nnz + 1, T2_ERR_INVALID_ARG, "mel filters are not contiguous in frequency");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  T2_CHECK_CUDA(cudaMemcpyAsync(d_plan, h.data(), p.bytes, cudaMemcpyHostToDevice, st));
  T2_CHECK_CUDA(cudaStreamSynchronize(st));
  return T2_OK;
}

extern "C" int t2_stft_mel_frames(const t2_audio_config_t* cfg, int n_samples) {
  return cfg ? 1 + n_samples / cfg->hop_size : 0;  // librosa centre=True: 1 + len // hop
}

extern "C" int t2_stft_mel_f32(const t2_audio_config_t* cfg, const void* d_plan, const float* d_wav, int B,
                               int n_samples, float preemphasis, float gain, float* d_mel, float* d_linear,
                               int time_major, void* stream) {
  Plan p;
  int rc = make_plan(cfg, p, nullptr);
  if (rc) return rc;
  T2_REQUIRE(d_plan && d_wav && d_mel && B >= 1 && n_samples >= 1, T2_ERR_INVALID_ARG, "stft_mel: bad arguments");
  const StftArgs a = stft_args(cfg, p, d_plan, d_wav, B, n_samples, preemphasis, gain, d_mel, d_linear, time_major);
  const int sms = device_sms();
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  rc = by_nfft(cfg->n_fft, [&](auto n) { return launch_stft_mel<decltype(n)::value>(a, sms, st); });
  if (rc) return rc;
  T2_CHECK_CUDA(cudaGetLastError());
  return T2_OK;
}

extern "C" int t2_mel_basis_f64(const t2_audio_config_t* cfg, double* h_basis) {
  Plan p;
  std::vector<double> W;
  int rc = make_plan(cfg, p, &W);
  if (rc) return rc;
  T2_REQUIRE(h_basis != nullptr, T2_ERR_INVALID_ARG, "mel_basis: null output");
  memcpy(h_basis, W.data(), W.size() * sizeof(double));
  return T2_OK;
}

extern "C" int t2_griffin_lim_bytes(const t2_audio_config_t* cfg, int B, int frames, long long* bytes) {
  T2_REQUIRE(cfg && bytes && B >= 1 && frames >= 2, T2_ERR_INVALID_ARG, "griffin_lim_bytes: bad arguments");
  *bytes = al((long long)B * frames * (cfg->n_fft / 2 + 1) * 8) + al((long long)B * frames * cfg->win_size * 4);
  return T2_OK;
}

extern "C" int t2_griffin_lim_f32(const t2_audio_config_t* cfg, const void* d_plan, const float* d_mag, float* d_phase_io, int B, int frames,
                                  int iters, unsigned long long seed, void* d_workspace, float* d_wav, void* stream) {
  Plan p;
  int rc = make_plan(cfg, p, nullptr);
  if (rc) return rc;
  T2_REQUIRE(d_plan && d_mag && d_workspace && d_wav && B >= 1 && frames >= 2 && iters >= 0, T2_ERR_INVALID_ARG, "griffin_lim: bad arguments");
  uint8_t* ws = static_cast<uint8_t*>(d_workspace);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  GlArgs a = gl_args(cfg, p, d_plan, B, frames);
  a.mag = d_mag;
  a.phase = d_phase_io ? reinterpret_cast<float2*>(d_phase_io) : reinterpret_cast<float2*>(ws);
  a.fr = reinterpret_cast<float*>(ws + al((long long)B * frames * (cfg->n_fft / 2 + 1) * 8));
  a.y = d_wav;
  const int sms = device_sms();
  const bool init_phase = d_phase_io == nullptr;
  rc = by_nfft(cfg->n_fft, [&](auto n) { return launch_griffin_lim<decltype(n)::value>(a, iters, init_phase, seed, sms, st); });
  if (rc) return rc;
  T2_CHECK_CUDA(cudaGetLastError());
  return T2_OK;
}

extern "C" int t2_dbg_audio_kernel(const t2_audio_config_t* cfg, const t2_dbg_kernel_t* call, void* stream) {
  T2_REQUIRE(call != nullptr, T2_ERR_INVALID_ARG, "dbg_audio_kernel: null call");
  Plan p;
  int rc = make_plan(cfg, p, nullptr);
  if (rc) return rc;
  void* const* q = call->p;
  const long long* i = call->i;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  switch (call->kernel) {
    case T2_DBG_AUDIO_STFT_MEL: {
      T2_REQUIRE(q[0] && q[1] && q[2], T2_ERR_INVALID_ARG, "dbg_audio_kernel STFT_MEL: null plan, wav or mel");
      T2_REQUIRE(in_range(i[0], 1, 65535) && in_range(i[1], 1, 1 << 30), T2_ERR_UNSUPPORTED_SHAPE,
                 "dbg_audio_kernel STFT_MEL: B must be in [1, 65535], n_samples in [1, 2^30]");
      T2_REQUIRE(in_range(i[2], 0, 1) && std::isfinite(call->f[0]) && std::isfinite(call->f[1]), T2_ERR_INVALID_ARG,
                 "dbg_audio_kernel STFT_MEL: time_major is 0 / 1, preemphasis and gain are finite");
      const StftArgs a = stft_args(cfg, p, q[0], static_cast<const float*>(q[1]), int(i[0]), int(i[1]), call->f[0], call->f[1],
                                   static_cast<float*>(q[2]), static_cast<float*>(q[3]), int(i[2]));
      const int sms = device_sms();
      rc = by_nfft(cfg->n_fft, [&](auto n) { return launch_stft_mel<decltype(n)::value>(a, sms, st); });
      break;
    }
    case T2_DBG_AUDIO_GL_INIT_PHASE:
      T2_REQUIRE(q[0] && in_range(i[0], 1, 1LL << 36), T2_ERR_INVALID_ARG, "dbg_audio_kernel GL_INIT_PHASE: null phase or n outside [1, 2^36]");
      launch_gl_init_phase(static_cast<float2*>(q[0]), i[0], call->seed, st);
      break;
    case T2_DBG_AUDIO_GL_ISTFT:
    case T2_DBG_AUDIO_GL_OLA:
    case T2_DBG_AUDIO_GL_STFT: {
      const int id = call->kernel;
      const char* what = id == T2_DBG_AUDIO_GL_ISTFT ? "GL_ISTFT" : id == T2_DBG_AUDIO_GL_OLA ? "GL_OLA" : "GL_STFT";
      T2_REQUIRE(q[0] && q[1] && q[2] && (id != T2_DBG_AUDIO_GL_ISTFT || q[3]), T2_ERR_INVALID_ARG, "dbg_audio_kernel %s: null pointer argument",
                 what);
      T2_REQUIRE(in_range(i[0], 1, 65535) && in_range(i[1], 2, 1 << 24) && (long long)cfg->hop_size * (i[1] - 1) < (1LL << 31),
                 T2_ERR_UNSUPPORTED_SHAPE, "dbg_audio_kernel %s: B must be in [1, 65535], frames in [2, 2^24], hop (frames - 1) < 2^31", what);
      GlArgs a = gl_args(cfg, p, q[0], int(i[0]), int(i[1]));
      const int sms = device_sms();
      if (id == T2_DBG_AUDIO_GL_ISTFT) {
        a.mag = static_cast<const float*>(q[1]); a.phase = static_cast<float2*>(q[2]); a.fr = static_cast<float*>(q[3]);
        rc = by_nfft(cfg->n_fft, [&](auto n) { return launch_gl_istft<decltype(n)::value>(a, sms, st); });
      } else if (id == T2_DBG_AUDIO_GL_OLA) {
        a.fr = static_cast<float*>(q[1]); a.y = static_cast<float*>(q[2]);
        launch_gl_ola(a, st);
      } else {
        a.y = static_cast<float*>(q[1]); a.phase = static_cast<float2*>(q[2]);
        rc = by_nfft(cfg->n_fft, [&](auto n) { return launch_gl_stft<decltype(n)::value>(a, sms, st); });
      }
      break;
    }
    default:
      return t2_set_error(T2_ERR_INVALID_ARG, "dbg_audio_kernel: unknown kernel id %d", call->kernel);
  }
  if (rc) return rc;
  T2_CHECK_CUDA(cudaGetLastError());
  return T2_OK;
}

extern "C" int t2_preemphasis_f32(const float* d_x, float* d_y, int B, int n_samples, float k, void* stream) {
  const long long n = (long long)B * n_samples;
  T2_REQUIRE(d_x && d_y && n > 0, T2_ERR_INVALID_ARG, "preemphasis: bad arguments");
  preemphasis_kernel<<<nblk(n), 256, 0, static_cast<cudaStream_t>(stream)>>>(d_x, d_y, n_samples, n, k); t2_count_launch();
  T2_CHECK_CUDA(cudaGetLastError());
  return T2_OK;
}
#define T2_ELTWISE(NAME, KERNEL, TIN, TOUT)                                                       \
  extern "C" int NAME(const TIN* d_in, TOUT* d_out, long long n, void* stream) {                  \
    T2_REQUIRE(d_in && d_out && n >= 0, T2_ERR_INVALID_ARG, #NAME ": bad arguments");             \
    if (n == 0) return T2_OK;                                                                     \
    KERNEL<<<nblk(n), 256, 0, static_cast<cudaStream_t>(stream)>>>(d_in, d_out, n); t2_count_launch();               \
    T2_CHECK_CUDA(cudaGetLastError());                                                            \
    return T2_OK;                                                                                 \
  }
T2_ELTWISE(t2_mulaw_quantize_f32_i32, mulaw_quantize_kernel, float, int)
T2_ELTWISE(t2_inv_mulaw_quantize_i32_f32, inv_mulaw_quantize_kernel, int, float)
T2_ELTWISE(t2_mulaw_f32, mulaw_kernel, float, float)
T2_ELTWISE(t2_inv_mulaw_f32, inv_mulaw_kernel, float, float)
