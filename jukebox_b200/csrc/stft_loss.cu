// Fused STFT magnitude comparison for the VQ-VAE's spectral losses (jukebox/utils/audio_utils.py:80-131).
//
// Per clip: resid = sum (|STFT a| - |STFT b|)^2 and norm_a = sum |STFT a|^2 over frames and onesided bins, with
// torch.stft's framing (center, reflect padding of n_fft / 2, window of win_length centred in n_fft).  No spectrogram
// reaches HBM: a CTA owns a run of F consecutive frames of one clip, stages the window support of that run once in
// shared memory (reflect padding by index arithmetic), and per group of frames
//   loads z = w * (a + i b) (one complex frame carries both signals),
//   runs an in-place radix-2^2 decimation-in-frequency FFT in shared memory (natural order in, bit-reversed out),
//   separates X_a[k] = (Z[k] + conj Z[N-k]) / 2, X_b[k] = (Z[k] - conj Z[N-k]) / 2i and accumulates the two sums.
// Sums: fp32 per thread and frame group, fp64 per thread across groups, a fixed shuffle tree per CTA into the caller's
// workspace, then a fixed-order sum over the CTAs of each clip.  The frame-to-CTA split depends on (T, n_fft, hop) only,
// so a clip's result has the same bits alone or in any batch.
#include "common.cuh"
#include "../../include/jkb200.h"

namespace {

constexpr int kThreads = 512;
constexpr int kFrameFloats = 4096;        // complex points per frame group: B = 4096 / n_fft frames
constexpr int kSpanFloats = 6656;         // staged samples per signal: F = (kSpanFloats - n_fft) / hop + 1 frames per CTA
constexpr int kTwiddles = 2730;           // per-stage twiddle tables of the largest FFT (sum of 2 m over m = 1024, 256, .., 1)
constexpr size_t kSmemBytes = sizeof(float2) * (kFrameFloats + kTwiddles) + sizeof(float) * 2 * kSpanFloats +
                              sizeof(double) * 2 * (kThreads / 32);

struct Plan {
    int64_t frames;          // 1 + T / hop
    int frames_per_cta;      // F
    int64_t ctas_per_clip;
};

bool is_pow2_fft(int n_fft) { return n_fft >= 256 && n_fft <= 4096 && (n_fft & (n_fft - 1)) == 0; }

Plan plan(int64_t T, int n_fft, int hop) {
    Plan p;
    p.frames = 1 + T / hop;
    const int B = kFrameFloats / n_fft;
    int64_t F = (kSpanFloats - n_fft) / hop + 1;
    if (F >= B) F -= F % B;                  // whole frame groups
    p.frames_per_cta = (int)F;
    p.ctas_per_clip = (p.frames + F - 1) / F;
    return p;
}

__device__ __forceinline__ float2 cmul(float2 a, float2 b) { return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }
__device__ __forceinline__ float2 cadd(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 csub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
__device__ __forceinline__ float2 mul_negi(float2 a) { return make_float2(a.y, -a.x); }

__device__ __forceinline__ int64_t reflect(int64_t i, int64_t T) { return i < 0 ? -i : (i >= T ? 2 * (T - 1) - i : i); }

__global__ void __launch_bounds__(kThreads, 2)
stft_mag_diff_kernel(const float* __restrict__ a, const float* __restrict__ b, const float* __restrict__ window,
                     double* __restrict__ partials, int64_t T, int log_n, int hop, int win_length, int frames_per_cta,
                     int64_t frames) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float2* z = reinterpret_cast<float2*>(smem_raw);
    float2* tw = z + kFrameFloats;
    float* sa = reinterpret_cast<float*>(tw + kTwiddles);
    float* sb = sa + kSpanFloats;
    double* red = reinterpret_cast<double*>(sb + kSpanFloats);

    const int N = 1 << log_n, B = kFrameFloats >> log_n, tid = threadIdx.x;
    const int left = (N - win_length) / 2;
    const int64_t clip = blockIdx.y;
    const int64_t f0 = (int64_t)blockIdx.x * frames_per_cta;
    const int nf = frames - f0 < frames_per_cta ? (int)(frames - f0) : frames_per_cta;

    // twiddles of every radix-2^2 stage, contiguous per stage: [W_4m^j, j < m | W_2m^j, j < m], from sincospi in fp64
    for (int m = N >> 2, off = 0; m >= 1; off += 2 * m, m >>= 2) {
        for (int j = tid; j < m; j += kThreads) {
            double s, c;
            sincospi(2.0 * j / (4.0 * m), &s, &c);
            tw[off + j] = make_float2((float)c, (float)-s);
            sincospi(2.0 * j / (2.0 * m), &s, &c);
            tw[off + m + j] = make_float2((float)c, (float)-s);
        }
    }
    // window support of the CTA's frames: padded position f * hop + left + i is signal sample f * hop - N/2 + left + i
    const int64_t s0 = f0 * hop - N / 2 + left;
    const int span = (nf - 1) * hop + win_length;
    const float* ac = a + clip * T;
    const float* bc = b + clip * T;
    for (int i = tid; i < span; i += kThreads) {
        const int64_t src = reflect(s0 + i, T);
        sa[i] = __ldg(ac + src);
        sb[i] = __ldg(bc + src);
    }
    __syncthreads();

    double acc_r = 0.0, acc_n = 0.0;
    const int half = N >> 1;
    for (int g0 = 0; g0 < nf; g0 += B) {
        for (int e = tid; e < kFrameFloats; e += kThreads) {
            const int fl = g0 + (e >> log_n), j = (e & (N - 1)) - left;
            float2 v = make_float2(0.f, 0.f);
            if (fl < nf && j >= 0 && j < win_length) {
                const float w = __ldg(window + j);
                const int o = fl * hop + j;
                v = make_float2(w * sa[o], w * sb[o]);
            }
            z[e] = v;
        }
        __syncthreads();
        int off = 0;
        for (int m = N >> 2; m >= 1; off += 2 * m, m >>= 2) {
            const int q = N >> 2;
            for (int t = tid; t < B * q; t += kThreads) {
                const int fb = t >> (log_n - 2), r = t & (q - 1);
                const int j = r & (m - 1);
                float2* p = z + (fb << log_n) + ((r - j) << 2) + j;
                const float2 x0 = p[0], x1 = p[m], x2 = p[2 * m], x3 = p[3 * m];
                const float2 w4 = tw[off + j], w2 = tw[off + m + j];
                const float2 y0 = cadd(x0, x2), y2 = cmul(csub(x0, x2), w4);
                const float2 y1 = cadd(x1, x3), y3 = cmul(mul_negi(csub(x1, x3)), w4);
                p[0] = cadd(y0, y1);
                p[m] = cmul(csub(y0, y1), w2);
                p[2 * m] = cadd(y2, y3);
                p[3 * m] = cmul(csub(y2, y3), w2);
            }
            __syncthreads();
        }
        if (log_n & 1) {                    // odd log2 n_fft: one radix-2 stage of span 1 is left
            for (int t = tid; t < kFrameFloats / 2; t += kThreads) {
                float2* p = z + 2 * t;
                const float2 u = p[0], v = p[1];
                p[0] = cadd(u, v);
                p[1] = csub(u, v);
            }
            __syncthreads();
        }
        // position p holds Z[bitrev(p)]; onesided bin k < N/2 sits at an even position, bin N/2 at position 1
        float sr = 0.f, sn = 0.f;
        const int bins = half + 1;
        for (int e = tid; e < B * bins; e += kThreads) {
            const int fb = e / bins, i = e - fb * bins;
            const int p = i < half ? 2 * i : 1;
            const int k = __brev(p) >> (32 - log_n);
            const int pq = __brev((N - k) & (N - 1)) >> (32 - log_n);
            const float2 zk = z[(fb << log_n) + p], zm = z[(fb << log_n) + pq];
            const float ar = 0.5f * (zk.x + zm.x), ai = 0.5f * (zk.y - zm.y);
            const float br = 0.5f * (zk.y + zm.y), bi = 0.5f * (zm.x - zk.x);
            const float pa = ar * ar + ai * ai;
            const float d = sqrtf(pa) - sqrtf(br * br + bi * bi);
            sr += d * d;
            sn += pa;
        }
        acc_r += sr;
        acc_n += sn;
        __syncthreads();
    }

#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        acc_r += __shfl_xor_sync(0xffffffffu, acc_r, o);
        acc_n += __shfl_xor_sync(0xffffffffu, acc_n, o);
    }
    if ((tid & 31) == 0) {
        red[2 * (tid >> 5)] = acc_r;
        red[2 * (tid >> 5) + 1] = acc_n;
    }
    __syncthreads();
    if (tid == 0) {
        double r = 0.0, n = 0.0;
        for (int w = 0; w < kThreads / 32; ++w) {
            r += red[2 * w];
            n += red[2 * w + 1];
        }
        double* out = partials + 2 * (clip * gridDim.x + blockIdx.x);
        out[0] = r;
        out[1] = n;
    }
}

// resid[n], norm_a[n] = the CTA partials of clip n summed in CTA order
__global__ void stft_reduce_kernel(const double* __restrict__ partials, double* __restrict__ resid,
                                   double* __restrict__ norm_a, int n, int64_t ctas) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= n) return;
    double r = 0.0, s = 0.0;
    for (int64_t i = 0; i < ctas; ++i) {
        r += partials[2 * (c * ctas + i)];
        s += partials[2 * (c * ctas + i) + 1];
    }
    resid[c] = r;
    norm_a[c] = s;
}

}  // namespace

extern "C" size_t jk_stft_workspace_bytes(int n, int64_t T, int n_fft, int hop) {
    if (n < 1 || T < 1 || hop < 1 || !is_pow2_fft(n_fft)) return 0;
    return sizeof(double) * 2 * (size_t)n * (size_t)plan(T, n_fft, hop).ctas_per_clip;
}

extern "C" int jk_stft_mag_diff(const float* a, const float* b, const float* window, double* resid, double* norm_a,
                                int n, int64_t T, int n_fft, int hop, int win_length, void* workspace,
                                size_t workspace_bytes, jk_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    JK_REQUIRE(a && b && window && resid && norm_a && workspace, "jk_stft_mag_diff: null argument");
    JK_REQUIRE(is_pow2_fft(n_fft), "jk_stft_mag_diff: n_fft %d must be a power of two in [256, 4096]", n_fft);
    JK_REQUIRE(win_length >= 1 && win_length <= n_fft, "jk_stft_mag_diff: win_length %d must be in [1, n_fft = %d]",
               win_length, n_fft);
    JK_REQUIRE(hop >= 1, "jk_stft_mag_diff: hop %d must be >= 1", hop);
    JK_REQUIRE(n >= 1 && n <= 65535, "jk_stft_mag_diff: n = %d clips must be in [1, 65535]", n);
    JK_REQUIRE(T > n_fft / 2, "jk_stft_mag_diff: reflect padding of n_fft / 2 = %d needs T > %d samples, got %lld",
               n_fft / 2, n_fft / 2, (long long)T);
    const Plan p = plan(T, n_fft, hop);
    JK_REQUIRE(p.ctas_per_clip <= 0x7fffffff, "jk_stft_mag_diff: T = %lld is too long", (long long)T);
    const size_t need = jk_stft_workspace_bytes(n, T, n_fft, hop);
    JK_REQUIRE(workspace_bytes >= need, "jk_stft_mag_diff: workspace of %zu bytes, %zu needed", workspace_bytes, need);

    if (int rc = jk::set_max_smem_once<stft_mag_diff_kernel>((int)kSmemBytes)) return rc;
    int log_n = 0;
    while ((1 << log_n) < n_fft) ++log_n;
    double* partials = static_cast<double*>(workspace);
    stft_mag_diff_kernel<<<dim3((unsigned)p.ctas_per_clip, (unsigned)n), kThreads, kSmemBytes, stream>>>(
        a, b, window, partials, T, log_n, hop, win_length, p.frames_per_cta, p.frames);
    JK_CHECK_CUDA(cudaGetLastError());
    stft_reduce_kernel<<<(n + 127) / 128, 128, 0, stream>>>(partials, resid, norm_a, n, p.ctas_per_clip);
    JK_CHECK_CUDA(cudaGetLastError());
    return 0;
}
