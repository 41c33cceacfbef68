// optim.cu -- the optimizer step on device (sm_90a): Adam over every tensor of a parameter group in one launch, then
// every cached weight packing of those parameters rebuilt in one launch.  Both launches take their whole descriptor
// table as ONE by-value kernel parameter (CUDA 12.1+ allows 32764 bytes on sm_70+), read in place through
// __grid_constant__, so a CUDA graph captures it with no host-to-device copy and the grads may sit at new addresses
// on every step.  A longer list is split into several launches of at most the table's capacity.
#include <cuda_bf16.h>

#include "common.cuh"
#include "pack.cuh"

namespace {

constexpr int NT = 256;
constexpr int ADAM_CHUNK = 4096;          // elements of one tensor per CTA iteration
constexpr int REPACK_CHUNK = 2048;        // elements of one packing per CTA iteration
constexpr int MAX_PARAM_BYTES = 32764;    // kernel parameter limit of CUDA 12.1+ on sm_70+
constexpr int ADAM_CAP = 480;             // tensors per vqb_adam_multi_f32 launch
constexpr int REPACK_CAP = 480;           // descriptors + step counters per vqb_repack_multi launch
constexpr int STEP_JOB = -1;              // a repack job that advances one step counter

struct AdamDesc {
    float *p;
    const float *g;
    float *m, *v, *vmax;
    const float *step;
    long long numel, chunk0;              // chunk0: the tensor's first chunk in the launch's concatenation
};

struct AdamTable {
    int n, amsgrad;
    double lr, beta1, beta2;              // the bias corrections are formed in double, as torch's Python scalars are
    float w1, b2, w2, eps, wd;            // 1 - beta1, beta2, 1 - beta2, eps, weight_decay rounded to fp32 once
    AdamDesc t[ADAM_CAP];
};
static_assert(sizeof(AdamTable) <= MAX_PARAM_BYTES, "Adam table exceeds the kernel parameter limit");

struct Job {
    void *dst;
    const float *src;
    long long chunk0;
    int layout, Cout, Cin, Cin_pad, kh, kw, transposed, rows, cols;
};

struct RepackTable {
    int n;
    Job j[REPACK_CAP];
};
static_assert(sizeof(RepackTable) <= MAX_PARAM_BYTES, "repack table exceeds the kernel parameter limit");

// index of the descriptor holding chunk c: the last one whose chunk0 <= c
template <typename D>
__device__ __forceinline__ int find_chunk(const D *d, int n, long long c) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (d[mid].chunk0 <= c) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// One element, in the order of torch's _single_tensor_adam with each of its tensor ops rounded as torch's CUDA kernels
// round them (one fused multiply-add where the kernel's expression is `a + alpha * b`):
//   grad.add(param, alpha=wd); exp_avg.lerp_(grad, 1 - beta1); exp_avg_sq.mul_(beta2).addcmul_(grad, grad, 1 - beta2);
//   amsgrad max; denom = (sqrt(v) / bc2_sqrt).add_(eps), the division by the scalar a product with its reciprocal,
//   formed in double and rounded to fp32; param.addcdiv_(exp_avg, denom, value=-lr / bc1).
__device__ __forceinline__ void adam_elem(float &p, float g, float &m, float &v, float &vm, bool ams,
                                          const AdamTable &t, float alpha, float inv_bc2) {
    if (t.wd != 0.f) g = __fmaf_rn(p, t.wd, g);
    const float d = __fsub_rn(g, m);
    m = t.w1 < 0.5f ? __fmaf_rn(t.w1, d, m) : __fmaf_rn(-d, __fsub_rn(1.f, t.w1), g);
    v = __fmaf_rn(t.w2, __fmul_rn(g, g), __fmul_rn(v, t.b2));
    float vh = v;
    if (ams) {
        vm = (vm > v || isnan(vm)) ? vm : v;      // torch.maximum: NaN propagates
        vh = vm;
    }
    const float denom = __fadd_rn(__fmul_rn(__fsqrt_rn(vh), inv_bc2), t.eps);
    p = __fmaf_rn(alpha, __fdiv_rn(m, denom), p);
}

__device__ __forceinline__ bool al16(const void *q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; }

__global__ void __launch_bounds__(NT) adam_kernel(const __grid_constant__ AdamTable t, long long chunks) {
    const bool ams = t.amsgrad != 0;
    for (long long c = blockIdx.x; c < chunks; c += gridDim.x) {
        const AdamDesc &d = t.t[find_chunk(t.t, t.n, c)];
        const long long e0 = (c - d.chunk0) * ADAM_CHUNK;
        const long long e1 = min(d.numel, e0 + ADAM_CHUNK);
        // the step this update takes: the counter (advanced by the repack launch after it) + 1, in fp32 as torch's
        // step_t += 1, then the bias corrections in double, each rounded to fp32 once
        const double s = (double)(__ldg(d.step) + 1.f);
        const double bc1 = 1.0 - pow(t.beta1, s), bc2 = 1.0 - pow(t.beta2, s);
        const float alpha = (float)(-(t.lr / bc1));
        const float inv_bc2 = (float)(1.0 / sqrt(bc2));
        long long i0 = e0;
        if (al16(d.p) && al16(d.g) && al16(d.m) && al16(d.v) && (!ams || al16(d.vmax))) {
            const long long n4 = (e1 - e0) >> 2;
            for (long long q = threadIdx.x; q < n4; q += NT) {
                const long long i = e0 + 4 * q;
                float4 p = *reinterpret_cast<float4 *>(d.p + i), m = *reinterpret_cast<float4 *>(d.m + i);
                float4 v = *reinterpret_cast<float4 *>(d.v + i);
                const float4 g = __ldg(reinterpret_cast<const float4 *>(d.g + i));
                float4 vm = ams ? *reinterpret_cast<float4 *>(d.vmax + i) : make_float4(0.f, 0.f, 0.f, 0.f);
                adam_elem(p.x, g.x, m.x, v.x, vm.x, ams, t, alpha, inv_bc2);
                adam_elem(p.y, g.y, m.y, v.y, vm.y, ams, t, alpha, inv_bc2);
                adam_elem(p.z, g.z, m.z, v.z, vm.z, ams, t, alpha, inv_bc2);
                adam_elem(p.w, g.w, m.w, v.w, vm.w, ams, t, alpha, inv_bc2);
                *reinterpret_cast<float4 *>(d.p + i) = p;
                *reinterpret_cast<float4 *>(d.m + i) = m;
                *reinterpret_cast<float4 *>(d.v + i) = v;
                if (ams) *reinterpret_cast<float4 *>(d.vmax + i) = vm;
            }
            i0 = e0 + 4 * n4;
        }
        for (long long i = i0 + threadIdx.x; i < e1; i += NT) {
            float p = d.p[i], m = d.m[i], v = d.v[i], vm = ams ? d.vmax[i] : 0.f;
            adam_elem(p, __ldg(d.g + i), m, v, vm, ams, t, alpha, inv_bc2);
            d.p[i] = p;
            d.m[i] = m;
            d.v[i] = v;
            if (ams) d.vmax[i] = vm;
        }
    }
}

__host__ __device__ long long job_elems(const Job &j) {
    switch (j.layout) {
        case VQB_PACK_F32:
        case VQB_PACK_BF16: return (long long)j.kh * j.kw * j.Cout * j.Cin_pad;
        case VQB_PACK_SHUFFLE_F32:
        case VQB_PACK_SHUFFLE_BF16: return 9LL * 16 * j.Cin;
        case VQB_PACK_PRIOR_F32: return (long long)j.rows * j.cols * j.Cin * j.Cout;
        case VQB_PACK_MASK_ZERO: return (long long)j.Cout * j.Cin * j.kh * j.kw;
        case VQB_PACK_PRIOR_PAD_F32:      // Cin_pad = Cp, transposed = kout + 4*kin (vqb_pack_layout)
            return (long long)j.rows * j.cols * pad_width(j.Cin, j.transposed >> 2, j.Cin_pad) *
                   pad_width(j.Cout, j.transposed & 3, j.Cin_pad);
        case VQB_PACK_PAD_F32:
            return (long long)pad_width(j.Cout, j.transposed & 3, j.Cin_pad) *
                   pad_width(j.Cin, j.transposed >> 2, j.Cin_pad) * j.kh * j.kw;
        case VQB_PACK_UNPAD_F32: return (long long)j.Cout * j.Cin * j.kh * j.kw;
        default: return 1;                // STEP_JOB
    }
}

__global__ void __launch_bounds__(NT) repack_kernel(const __grid_constant__ RepackTable t, long long chunks) {
    for (long long c = blockIdx.x; c < chunks; c += gridDim.x) {
        const Job &j = t.j[find_chunk(t.j, t.n, c)];
        const long long e0 = (c - j.chunk0) * REPACK_CHUNK;
        const long long e1 = min(job_elems(j), e0 + REPACK_CHUNK);
        for (long long i = e0 + threadIdx.x; i < e1; i += NT) {
            switch (j.layout) {
                case VQB_PACK_F32:
                    static_cast<float *>(j.dst)[i] = pack_kmajor_at(j.src, i, j.Cout, j.Cin, j.Cin_pad, j.kh, j.kw,
                                                                    j.transposed);
                    break;
                case VQB_PACK_BF16:
                    static_cast<__nv_bfloat16 *>(j.dst)[i] =
                        __nv_bfloat16(pack_kmajor_at(j.src, i, j.Cout, j.Cin, j.Cin_pad, j.kh, j.kw, j.transposed));
                    break;
                case VQB_PACK_SHUFFLE_F32:
                    static_cast<float *>(j.dst)[i] = pack_shuffle_at(j.src, (int)i, j.Cout, j.Cin);
                    break;
                case VQB_PACK_SHUFFLE_BF16:
                    static_cast<__nv_bfloat16 *>(j.dst)[i] = __nv_bfloat16(pack_shuffle_at(j.src, (int)i, j.Cout, j.Cin));
                    break;
                case VQB_PACK_PRIOR_F32:
                    static_cast<float *>(j.dst)[i] = pack_prior_at(j.src, i, j.Cout, j.Cin, j.kh, j.kw, j.cols);
                    break;
                case VQB_PACK_MASK_ZERO: {    // the parameter's taps outside rows x cols; no packing reads them
                    const int s = (int)(i % j.kw), r = (int)((i / j.kw) % j.kh);
                    if (r >= j.rows || s >= j.cols) static_cast<float *>(j.dst)[i] = 0.f;
                    break;
                }
                case VQB_PACK_PRIOR_PAD_F32:
                    static_cast<float *>(j.dst)[i] = pack_prior_pad_at(j.src, i, j.Cout, j.Cin, j.kh, j.kw, j.cols,
                                                                       j.Cin_pad, j.transposed & 3, j.transposed >> 2);
                    break;
                case VQB_PACK_PAD_F32:
                    static_cast<float *>(j.dst)[i] = pack_pad_at(j.src, i, j.Cout, j.Cin, j.kh * j.kw, j.Cin_pad,
                                                                 j.transposed & 3, j.transposed >> 2);
                    break;
                case VQB_PACK_UNPAD_F32:
                    static_cast<float *>(j.dst)[i] = unpad_at(j.src, i, j.Cout, j.Cin, j.kh * j.kw, j.Cin_pad,
                                                              j.transposed & 3, j.transposed >> 2);
                    break;
                default:                      // STEP_JOB: nothing in this launch reads the counter
                    *static_cast<float *>(j.dst) += 1.f;
                    break;
            }
        }
    }
}

unsigned grid_for_chunks(long long chunks) {
    const long long cap = 148LL * 8;
    return (unsigned)(chunks < cap ? chunks : cap);
}

bool bad_hyper(double lr, double beta1, double beta2, double eps, double wd) {
    return !(lr >= 0.0) || !(eps >= 0.0) || !(beta1 >= 0.0 && beta1 < 1.0) || !(beta2 >= 0.0 && beta2 < 1.0) ||
           !(wd >= 0.0);
}

// the padded layouts' geometry (vqb_pack_layout): Cin_pad = Cp > 0, transposed = kout + 4*kin with kinds 0..2, at
// least one padded axis, a gate axis even, and no real channel count above its padded half
bool bad_axis(int n, int kind, int cp) {
    if (kind == 0) return false;
    return (kind == 2 && n % 2 != 0) || n / kind > cp;
}

bool bad_padding(const vqb_pack_desc &d) {
    const int kout = d.transposed & 3, kin = d.transposed >> 2;
    return !d.src || d.Cin_pad <= 0 || d.transposed < 1 || d.transposed > 10 || kout > 2 || kin > 2 ||
           bad_axis(d.Cout, kout, d.Cin_pad) || bad_axis(d.Cin, kin, d.Cin_pad);
}

bool bad_desc(const vqb_pack_desc &d) {
    if (!d.dst || d.Cout <= 0 || d.Cin <= 0 || d.kh <= 0 || d.kw <= 0) return true;
    switch (d.layout) {
        case VQB_PACK_F32:
        case VQB_PACK_BF16: return !d.src || d.Cin_pad < d.Cin || (d.transposed != 0 && d.transposed != 1);
        case VQB_PACK_SHUFFLE_F32:
        case VQB_PACK_SHUFFLE_BF16: return !d.src || d.kh != 4 || d.kw != 4 || d.Cout > 4;
        case VQB_PACK_PRIOR_F32:
        case VQB_PACK_MASK_ZERO:
            return (d.layout == VQB_PACK_PRIOR_F32 && !d.src) || d.rows < 0 || d.cols < 0 || d.rows > d.kh ||
                   d.cols > d.kw;
        case VQB_PACK_PRIOR_PAD_F32:
            if (d.rows < 0 || d.cols < 0 || d.rows > d.kh || d.cols > d.kw) return true;
            return bad_padding(d);
        case VQB_PACK_PAD_F32:
        case VQB_PACK_UNPAD_F32: return bad_padding(d);
        default: return true;
    }
}

}  // namespace

extern "C" int vqb_adam_capacity(void) { return ADAM_CAP; }
extern "C" int vqb_repack_capacity(void) { return REPACK_CAP; }

extern "C" int vqb_adam_multi_f32(const vqb_adam_tensor *tensors, int n, double lr, double beta1, double beta2,
                                  double eps, double weight_decay, int amsgrad, void *stream) {
    if (n < 0 || (n > 0 && !tensors) || bad_hyper(lr, beta1, beta2, eps, weight_decay)) return VQB_ERR_BAD_ARG;
    for (int i = 0; i < n; ++i) {
        const vqb_adam_tensor &x = tensors[i];
        if (!x.param || !x.grad || !x.exp_avg || !x.exp_avg_sq || !x.step || x.numel < 0 ||
            (amsgrad && !x.max_exp_avg_sq))
            return VQB_ERR_BAD_ARG;
    }
    AdamTable t;                          // ~30 KB on the host stack, copied into the launch
    t.amsgrad = amsgrad != 0;
    t.lr = lr, t.beta1 = beta1, t.beta2 = beta2;
    t.w1 = (float)(1.0 - beta1), t.b2 = (float)beta2, t.w2 = (float)(1.0 - beta2);
    t.eps = (float)eps, t.wd = (float)weight_decay;
    int i = 0;
    while (i < n) {
        t.n = 0;
        long long chunks = 0;
        for (; i < n && t.n < ADAM_CAP; ++i) {
            const vqb_adam_tensor &x = tensors[i];
            if (x.numel == 0) continue;
            t.t[t.n++] = AdamDesc{x.param, x.grad, x.exp_avg, x.exp_avg_sq, amsgrad ? x.max_exp_avg_sq : nullptr,
                                  x.step, (long long)x.numel, chunks};
            chunks += (x.numel + ADAM_CHUNK - 1) / ADAM_CHUNK;
        }
        if (!chunks) continue;
        adam_kernel<<<grid_for_chunks(chunks), NT, 0, (cudaStream_t)stream>>>(t, chunks);
        VQB_COUNT_LAUNCH(1);
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return vqb_cuda_status(e);
    }
    return 0;
}

extern "C" int vqb_repack_multi(const vqb_pack_desc *descs, int n, float *const *steps, int n_steps, void *stream) {
    if (n < 0 || n_steps < 0 || (n > 0 && !descs) || (n_steps > 0 && !steps)) return VQB_ERR_BAD_ARG;
    for (int i = 0; i < n; ++i)
        if (bad_desc(descs[i])) return VQB_ERR_BAD_ARG;
    for (int i = 0; i < n_steps; ++i)
        if (!steps[i]) return VQB_ERR_BAD_ARG;
    RepackTable t;
    int i = 0;                           // descriptors first, then the step counters, REPACK_CAP jobs per launch
    while (i < n + n_steps) {
        t.n = 0;
        long long chunks = 0;
        for (; i < n + n_steps && t.n < REPACK_CAP; ++i) {
            Job j{};
            if (i < n) {
                const vqb_pack_desc &d = descs[i];
                j = Job{d.dst, d.src, 0, d.layout, d.Cout, d.Cin, d.Cin_pad, d.kh, d.kw, d.transposed, d.rows, d.cols};
            } else {
                j.dst = steps[i - n];
                j.layout = STEP_JOB;
            }
            const long long e = job_elems(j);
            if (e == 0) continue;
            j.chunk0 = chunks;
            t.j[t.n++] = j;
            chunks += (e + REPACK_CHUNK - 1) / REPACK_CHUNK;
        }
        if (!chunks) continue;
        repack_kernel<<<grid_for_chunks(chunks), NT, 0, (cudaStream_t)stream>>>(t, chunks);
        VQB_COUNT_LAUNCH(1);
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return vqb_cuda_status(e);
    }
    return 0;
}
