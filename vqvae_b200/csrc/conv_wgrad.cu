// conv_wgrad.cu -- weight and bias gradient of one nn.Conv2d / nn.ConvTranspose2d layer, fp32 on CUDA cores (sm_90a).
//
// Both kinds are one product reduced over the positions of an "iterated" grid X, against the other operand Y read at
// each tap's shifted position  y = x * stride - pad + (r, s)  (zero outside Y's grid):
//   Conv2d           X = g_out (the output grid), Y = in     ->  dW[co][ci][r][s], the (Cout, Cin, kh, kw) parameter
//   ConvTranspose2d  X = in    (the input grid),  Y = g_out  ->  dW[ci][co][r][s], the (Cin, Cout, kh, kw) parameter
// Rows are X's channels and columns tap * Cy + cy, so the reduction writes dW in the parameter's own layout.  The bias
// gradient sums g_out over its own grid: for a Conv2d it is a column of ones after the tap columns; a ConvTranspose2d
// iterates over the input grid, so its bias is a second, one-column product with X = g_out.
// The products run on the FFMA GEMM the prior's backward also uses (ffma_gemm.cuh), with X and the tap-shifted Y as
// its operands: both stage four channels at a time with one float4 load when the channels are contiguous.  The
// positions are split into fixed chunks whose partials are summed in chunk order: no atomics, so two calls give
// bitwise-equal gradients.
#include "ffma_gemm.cuh"

namespace {

struct Act {                       // a (B, C, H, W) activation addressed through element strides
    const float *p;
    int C, H, W;
    long long sn, sh, sw, sc;
    bool vec;                      // channels contiguous, C % 4 == 0, 16-byte aligned: float4 along the channels
    __device__ __forceinline__ const float *at(long long b, int y, int x) const { return p + b * sn + y * sh + x * sw; }
};

struct Job {
    Act x, y;
    int kw, taps, stride, pad;
    int ycols, cols;               // columns read from Y (taps * y.C); a column of ones follows when cols > ycols
    long long P;                   // positions of X's grid
    WgradSplit sp;
    float *part;                   // [sp.splits][x.C][cols]
};

struct Pos {                       // position p of a (B, H, W) grid
    long long b;
    int y, x;
    __device__ __forceinline__ Pos(long long p, int H, int W) {
        const long long hw = (long long)H * W;
        b = p / hw;
        const int rem = (int)(p - b * hw);
        y = rem / W;
        x = rem - y * W;
    }
};

// X as the A operand: row c = channel c, k = position p of X's grid
struct XGrid {
    Act x;
    bool j_fast, vec;              // positions fast when the channels are not contiguous; vec: x.vec
    __device__ __forceinline__ const float *at(long long p) const {
        const Pos q(p, x.H, x.W);
        return x.at(q.b, q.y, q.x);
    }
    __device__ __forceinline__ float operator()(int c, long long p) const { return __ldg(at(p) + c * x.sc); }
    __device__ __forceinline__ float4 four(int c, long long p) const {
        return __ldg(reinterpret_cast<const float4 *>(at(p) + c));
    }
};

// Y at the taps as the B operand: k = position p = (b, oy, ox) of X's grid (H x W), column n = tap * C + c reads channel
// c of Y at (oy * stride - pad + r, ox * stride - pad + s), tap = r * kw + s; 0 outside Y's grid
struct YTap {
    Act y;
    int H, W, kw, stride, pad;
    bool j_fast, vec;              // columns fast when the channels are contiguous; vec: y.vec (C % 4 == 0, so a group
                                   // of four columns stays inside one tap)
    // tap `tap` of position p in Y, or nullptr outside Y's grid
    __device__ __forceinline__ const float *at(long long p, int tap) const {
        const int r = tap / kw, s = tap - r * kw;
        const Pos q(p, H, W);
        const int iy = q.y * stride - pad + r, ix = q.x * stride - pad + s;
        return iy < 0 || iy >= y.H || ix < 0 || ix >= y.W ? nullptr : y.at(q.b, iy, ix);
    }
    __device__ __forceinline__ float operator()(long long p, int n) const {
        const int tap = n / y.C, c = n - tap * y.C;
        const float *a = at(p, tap);
        return a ? __ldg(a + c * y.sc) : 0.f;
    }
    __device__ __forceinline__ float4 four(long long p, int n) const {
        const int tap = n / y.C, c = n - tap * y.C;
        const float *a = at(p, tap);
        return a ? __ldg(reinterpret_cast<const float4 *>(a + c)) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
};

// ---- host side ---------------------------------------------------------------------------------------------------
Act act(const float *p, int layout, int C, int H, int W) {
    Act a;
    a.p = p; a.C = C; a.H = H; a.W = W;
    layout_strides(layout, C, H, W, a.sn, a.sh, a.sw, a.sc);
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
        const XGrid a{j.x, j.x.sc != 1, j.x.vec};
        const WithOnes<YTap> b{YTap{j.y, j.x.H, j.x.W, j.kw, j.stride, j.pad, j.y.sc == 1, j.y.vec}, j.ycols};
        gemm(st, a, b, Partial{j.part, j.x.C, j.cols}, j.x.C, j.cols, j.P, j.sp);
        // partial columns tap * Cy + cy -> dW[row][cy][tap]; the ones column -> dbias[row]
        rj.j[i] = RJob{j.part, dW, dbias, j.x.C, j.y.C, j.taps, j.cols, j.sp.splits};
        most = most > (long long)j.x.C * j.cols ? most : (long long)j.x.C * j.cols;
    }
    wgrad_reduce(st, rj, n, most);
    VQB_COUNT_LAUNCH(n + 1);
    return vqb_cuda_status(cudaGetLastError());
}
