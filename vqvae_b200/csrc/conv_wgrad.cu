// conv_wgrad.cu -- weight and bias gradient of one nn.Conv2d / nn.ConvTranspose2d layer, fp32 on CUDA cores (sm_90a).
//
// Both kinds are one product reduced over the positions of an "iterated" grid X, against the other operand Y read at
// each tap's shifted position  y = x * stride - pad + (r, s)  (zero outside Y's grid):
//   Conv2d           X = g_out (the output grid), Y = in     ->  dW[co][ci][r][s], the (Cout, Cin, kh, kw) parameter
//   ConvTranspose2d  X = in    (the input grid),  Y = g_out  ->  dW[ci][co][r][s], the (Cin, Cout, kh, kw) parameter
// Rows are X's channels and columns tap * Cy + cy, so the reduction writes dW in the parameter's own layout.  The bias
// gradient sums g_out over its own grid: for a Conv2d it is a column of ones after the tap columns; a ConvTranspose2d
// iterates over the input grid, so its bias is a second, one-column product with X = g_out.
// Per CTA: a 64 x 64 tile of (rows x columns) over one chunk of positions, 16 positions per step staged in shared
// memory (float4 loads along the channel dimension when it is contiguous), 4 x 4 outputs per thread, each one fmaf
// chain in position order.  The chunk partials are summed in chunk order (wgrad_reduce.cuh): no atomics, so two calls
// give bitwise-equal gradients.
#include "wgrad_reduce.cuh"

namespace {

constexpr int BM = 64, BN = 64, BK = 16, GT = 256;        // CTA tile, positions per step, threads (16 x 16, 4 x 4 each)

struct Act {                       // a (B, C, H, W) activation addressed through element strides
    const float *p;
    int C, H, W;
    long long sn, sh, sw, sc;
    bool vec;                      // channels contiguous, C % 4 == 0, 16-byte aligned: float4 along the channels
};

struct Job {
    Act x, y;
    int kw, taps, stride, pad;
    int ycols, cols;               // columns read from Y (taps * y.C); a column of ones follows when cols > ycols
    long long P;                   // positions of X's grid
    WgradSplit sp;
    float *part;                   // [sp.splits][x.C][cols]
};

__device__ __forceinline__ void split_pos(long long p, int H, int W, long long &b, int &r, int &c) {
    const long long hw = (long long)H * W;
    b = p / hw;
    const int rem = (int)(p - b * hw);
    r = rem / W;
    c = rem - r * W;
}

__global__ void __launch_bounds__(GT) wgrad_kernel(const Job J) {
    __shared__ __align__(16) float Xs[BK][BM + 4];
    __shared__ __align__(16) float Ys[BK][BN + 4];
    const int tid = threadIdx.x, tm = tid / 16, tn = tid % 16;
    const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
    const long long p_begin = (long long)blockIdx.z * J.sp.chunk;
    const long long p_end = p_begin + J.sp.chunk < J.P ? p_begin + J.sp.chunk : J.P;
    const Act &X = J.x, &Y = J.y;
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

    // Y's element (position p, column n): channel n % Cy of tap n / Cy at p's shifted position, or the ones column
    auto y_at = [&](long long p, int n) -> float {
        if (p >= p_end || n >= J.cols) return 0.f;
        if (n >= J.ycols) return 1.f;
        const int tap = n / Y.C, c = n - tap * Y.C, r = tap / J.kw, s = tap - r * J.kw;
        long long b;
        int oy, ox;
        split_pos(p, X.H, X.W, b, oy, ox);
        const int iy = oy * J.stride - J.pad + r, ix = ox * J.stride - J.pad + s;
        if (iy < 0 || iy >= Y.H || ix < 0 || ix >= Y.W) return 0.f;
        return __ldg(Y.p + b * Y.sn + iy * Y.sh + ix * Y.sw + c * Y.sc);
    };

    for (long long p0 = p_begin; p0 < p_end; p0 += BK) {
        if (X.vec) {                                   // one float4 of channels per thread
            const int kk = tid / 16, mm = (tid % 16) * 4, m = m0 + mm;
            const long long p = p0 + kk;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (p < p_end && m < X.C) {
                long long b;
                int yy, xx;
                split_pos(p, X.H, X.W, b, yy, xx);
                v = __ldg(reinterpret_cast<const float4 *>(X.p + b * X.sn + yy * X.sh + xx * X.sw + m));
            }
            *reinterpret_cast<float4 *>(&Xs[kk][mm]) = v;
        } else {                                       // consecutive threads: consecutive addresses
            const bool cfast = X.sc == 1;
#pragma unroll
            for (int q = 0; q < BM * BK / GT; ++q) {
                const int e = tid + q * GT;
                const int mm = cfast ? e % BM : e / BK, kk = cfast ? e / BM : e % BK, m = m0 + mm;
                const long long p = p0 + kk;
                float v = 0.f;
                if (p < p_end && m < X.C) {
                    long long b;
                    int yy, xx;
                    split_pos(p, X.H, X.W, b, yy, xx);
                    v = __ldg(X.p + b * X.sn + yy * X.sh + xx * X.sw + m * X.sc);
                }
                Xs[kk][mm] = v;
            }
        }
        if (Y.vec) {                                   // four consecutive columns of one tap per thread
            const int kk = tid / 16, nn = (tid % 16) * 4, n = n0 + nn;
            const long long p = p0 + kk;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (n + 3 < J.ycols) {
                if (p < p_end) {
                    const int tap = n / Y.C, c = n - tap * Y.C, r = tap / J.kw, s = tap - r * J.kw;
                    long long b;
                    int oy, ox;
                    split_pos(p, X.H, X.W, b, oy, ox);
                    const int iy = oy * J.stride - J.pad + r, ix = ox * J.stride - J.pad + s;
                    if (iy >= 0 && iy < Y.H && ix >= 0 && ix < Y.W)
                        v = __ldg(reinterpret_cast<const float4 *>(Y.p + b * Y.sn + iy * Y.sh + ix * Y.sw + c));
                }
            } else {
                v = make_float4(y_at(p, n), y_at(p, n + 1), y_at(p, n + 2), y_at(p, n + 3));
            }
            *reinterpret_cast<float4 *>(&Ys[kk][nn]) = v;
        } else {
            const bool cfast = Y.sc == 1;
#pragma unroll
            for (int q = 0; q < BN * BK / GT; ++q) {
                const int e = tid + q * GT;
                const int nn = cfast ? e % BN : e / BK, kk = cfast ? e / BN : e % BK;
                Ys[kk][nn] = y_at(p0 + kk, n0 + nn);
            }
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < BK; ++kk) {
            const float4 av = *reinterpret_cast<const float4 *>(&Xs[kk][tm * 4]);
            const float4 bv = *reinterpret_cast<const float4 *>(&Ys[kk][tn * 4]);
            const float ar[4] = {av.x, av.y, av.z, av.w}, br[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(ar[i], br[j], acc[i][j]);
        }
        __syncthreads();
    }
    float *part = J.part + (long long)blockIdx.z * X.C * J.cols;
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int m = m0 + tm * 4 + i, n = n0 + tn * 4 + j;
            if (m < X.C && n < J.cols) part[(long long)m * J.cols + n] = acc[i][j];
        }
}

// ---- host side ---------------------------------------------------------------------------------------------------
Act act(const float *p, int layout, int C, int H, int W) {
    Act a;
    a.p = p; a.C = C; a.H = H; a.W = W;
    if (layout == VQB_NCHW) {
        a.sn = (long long)C * H * W; a.sc = (long long)H * W; a.sh = W; a.sw = 1;
    } else {
        a.sn = (long long)H * W * C; a.sh = (long long)W * C; a.sw = C; a.sc = 1;
    }
    a.vec = a.sc == 1 && C % 4 == 0 && (reinterpret_cast<uintptr_t>(p) & 15) == 0;
    return a;
}

Job make_job(const Act &x, const Act &y, int B, int kw, int taps, int stride, int pad, bool ones) {
    Job j;
    j.x = x; j.y = y;
    j.kw = kw; j.taps = taps; j.stride = stride; j.pad = pad;
    j.ycols = taps * y.C;
    j.cols = j.ycols + (ones ? 1 : 0);
    j.P = (long long)B * x.H * x.W;
    // the split follows the tap columns only, so a layer's dW is reduced in the same chunks with or without its bias,
    // and the plan with the ones column never needs fewer partials than the one without
    j.sp = wgrad_split(x.C, j.ycols > 0 ? j.ycols : j.cols, j.P, BM, BN, BK);
    j.part = nullptr;
    return j;
}

long long job_floats(const Job &j) { return (long long)j.sp.splits * j.x.C * j.cols; }

// The products of one layer (1, or 2 for a transposed conv with a bias) and `floats`, the partials they need; false
// when the geometry is bad.  Pointers may be null here: only the sizes are needed to size the workspace.  The plan
// with a bias needs at least as many partials as the one without (same splits, one more column or product).
bool plan(const float *in, const float *g_out, int B, int Cin, int H, int W, int Cout, int kh, int kw, int stride,
          int pad, int transposed, int in_layout, int gout_layout, bool bias, Job (&jobs)[2], int &n, long long &floats) {
    if (B <= 0 || Cin <= 0 || H <= 0 || W <= 0 || Cout <= 0 || kh <= 0 || kw <= 0 || stride <= 0 || pad < 0)
        return false;
    if ((in_layout != VQB_NCHW && in_layout != VQB_NHWC) || (gout_layout != VQB_NCHW && gout_layout != VQB_NHWC))
        return false;
    const ConvGeom g = conv_geom(kh, kw, stride, pad, transposed, H, W);
    if (g.OH <= 0 || g.OW <= 0) return false;
    const Act a_in = act(in, in_layout, Cin, H, W), a_g = act(g_out, gout_layout, Cout, g.OH, g.OW);
    if (transposed) {
        jobs[0] = make_job(a_in, a_g, B, kw, kh * kw, stride, pad, false);
        n = 1;
        if (bias) jobs[n++] = make_job(a_g, a_g, B, 1, 0, 1, 0, true);       // no tap columns: the ones column only
    } else {
        jobs[0] = make_job(a_g, a_in, B, kw, kh * kw, stride, pad, bias);
        n = 1;
    }
    floats = 0;
    for (int i = 0; i < n; ++i) floats += job_floats(jobs[i]);
    return true;
}

}  // namespace

extern "C" size_t vqb_conv_wgrad_workspace_bytes(int B, int Cin, int H, int W, int Cout, int kh, int kw, int stride,
                                                 int pad, int transposed) {
    Job jobs[2];
    int n;
    long long floats;
    if (!plan(nullptr, nullptr, B, Cin, H, W, Cout, kh, kw, stride, pad, transposed, VQB_NHWC, VQB_NHWC, true, jobs, n,
              floats))
        return 0;
    return (size_t)floats * sizeof(float);
}

extern "C" int vqb_conv_wgrad_f32(const float *in, const float *g_out, float *dW, float *dbias, int B, int Cin, int H,
                                  int W, int Cout, int kh, int kw, int stride, int pad, int transposed, int in_layout,
                                  int gout_layout, void *workspace, size_t workspace_bytes, void *stream) {
    if (!in || !g_out || !dW || !workspace) return VQB_ERR_BAD_ARG;
    Job jobs[2];
    int n;
    long long floats;
    if (!plan(in, g_out, B, Cin, H, W, Cout, kh, kw, stride, pad, transposed, in_layout, gout_layout, dbias != nullptr,
              jobs, n, floats))
        return VQB_ERR_BAD_ARG;
    if (workspace_bytes < (size_t)floats * sizeof(float)) return VQB_ERR_WORKSPACE;     // the partials this plan writes
    for (int i = 0; i < n; ++i)
        if (wgrad_cdiv(jobs[i].cols, BN) > 65535 || jobs[i].sp.splits > 65535) return VQB_ERR_UNSUPPORTED;
    cudaStream_t st = (cudaStream_t)stream;
    float *part = static_cast<float *>(workspace);
    RJobs rj;
    long long most = 0;
    for (int i = 0; i < n; ++i) {
        Job &j = jobs[i];
        j.part = part;
        part += job_floats(j);
        const dim3 grid(wgrad_cdiv(j.x.C, BM), wgrad_cdiv(j.cols, BN), j.sp.splits);
        wgrad_kernel<<<grid, GT, 0, st>>>(j);
        // partial columns tap * Cy + cy -> dW[row][cy][tap]; the ones column -> dbias[row]
        rj.j[i] = RJob{j.part, dW, dbias, j.x.C, j.y.C, j.taps, j.cols, j.sp.splits};
        most = most > (long long)j.x.C * j.cols ? most : (long long)j.x.C * j.cols;
    }
    wgrad_reduce(st, rj, n, most);
    VQB_COUNT_LAUNCH(n + 1);
    return vqb_cuda_status(cudaGetLastError());
}
