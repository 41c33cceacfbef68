// hconv.cu -- the bf16 pipeline's convolution layers (VQB_BF16 mode): weight packing plans and the entry points
// vqb_conv2d_bf16 / vqb_residual_layer_bf16, all computed by the wgmma implicit-GEMM kernel of wgconv.cu on bf16 NHWC
// activations with fp32 accumulation:
//   encoder.py:32-34  Conv2d k4 s2 p1          (taps read through stride-2 element strides of the input tensor map)
//   encoder.py:35-36  Conv2d k3 s1 p1
//   vqvae.py:16-17    Conv2d k1                 (fp32 output: z_e feeds the bit-exact VQ)
//   decoder.py:28-29  ConvTranspose2d k3 s1 p1
//   decoder.py:31-33  ConvTranspose2d k4 s2 p1  (four sub-pixel phases of 4 taps in one launch)
//   decoder.py:34-35  ConvTranspose2d k4 s2 p1 to <= 4 channels (one 3x3-neighbourhood GEMM, N = 16, pixel-shuffle
//                                                epilogue writing the NCHW fp32 module output)
//   residual.py:18-29 one ResidualLayer: 3x3 conv, ReLU and 1x1 conv chained inside one CTA per tile
// A packed weight is one 128-byte row of 64 bf16 input channels per (k-step, output column) in plan order, followed
// by the plan's row table (RowDesc per row); the kernel reads the rows of each k-step as one TMA box.
#include <cuda_bf16.h>

#include <cstdlib>
#include <cstring>
#include <vector>

#include "common.cuh"
#include "bf16_common.cuh"
#include "wgconv.h"

void convt_out_scatter_column(int n, int *co, int *ky, int *kx);

namespace {

constexpr int HC_MAX_STEPS = 40;      // per pass
constexpr int HC_MAX_CHUNKS = 8;

enum { ST_FIRST = 1, ST_NEWCHUNK = 2, ST_ENDCHUNK = 4, ST_HALFBOX = 8 };
enum { EPI_NHWC = 0, EPI_SHUFFLE_NCHW = 1 };

// ------------------------------------------------------------------------------------------------ host side: plans
struct RowDesc { int co, ci0, r, s; };          // one packed weight row = 64 input channels of (co, r, s); co < 0: zeros

struct PlanStep { int chunk, dy, dx, nb, d_col, w_row, flags; };

struct Plan {
    int kind = -1, Cin = 0, Cout = 0;
    int nchunks = 0, chunk_c0[HC_MAX_CHUNKS], chunk_p[HC_MAX_CHUNKS];
    int npass = 1, nsteps[2] = {0, 0};
    PlanStep steps[2][HC_MAX_STEPS];
    int NCOL = 0, nbmax = 0, nbhalf = 0, halo = 1, epi_mode = EPI_NHWC, cg = 0, sy = 1, sx = 1, transposed = 0, s2d = 0;
    std::vector<RowDesc> rows;
    int scatter_row0 = -1;          // VQB_CONVT_K4S2_OUT, Cin = 64, Cout = 3: first of the 64 GEMM-column rows of convt_out_bf16.cu
};

void add_step(Plan &pl, int pass, int chunk, int dy, int dx, int nb, int d_col, int w_row, bool half) {
    PlanStep &s = pl.steps[pass][pl.nsteps[pass]++];
    s.chunk = chunk; s.dy = dy; s.dx = dx; s.nb = nb; s.d_col = d_col; s.w_row = w_row; s.flags = half ? ST_HALFBOX : 0;
}

// returns false when the shape is outside what this kernel family covers
bool build_plan(Plan &pl, int kind, int Cin, int Cout) {
    pl = Plan();
    pl.kind = kind; pl.Cin = Cin; pl.Cout = Cout;
    if (kind == VQB_RES_W2_KIND) {
        // residual.py:23: 1x1 conv Cmid -> C; one K chunk, rows beyond Cin are zero (the pack kernel pads)
        if (Cin < 16 || Cin > 64 || Cin % 16 != 0 || Cout % 16 != 0 || Cout < 16 || Cout > 256) return false;
        pl.nchunks = 1; pl.chunk_c0[0] = 0; pl.chunk_p[0] = 0; pl.NCOL = Cout; pl.nbmax = Cout; pl.cg = Cout; pl.halo = 0;
        for (int c = 0; c < Cout; ++c) pl.rows.push_back({c, 0, 0, 0});
        pl.nsteps[0] = 1;
        PlanStep &st = pl.steps[0][0];
        st.chunk = 0; st.dy = 0; st.dx = 0; st.nb = Cout; st.d_col = 0; st.w_row = 0; st.flags = ST_FIRST | ST_NEWCHUNK | ST_ENDCHUNK;
        return true;
    }
    if (Cin % 64 != 0 || Cin < 64) return false;
    const int kc = Cin / 64;
    auto rows_for = [&](int co0, int nco, int ci0, int r, int s) {
        const int row0 = (int)pl.rows.size();
        for (int c = 0; c < nco; ++c) pl.rows.push_back({co0 + c, ci0, r, s});
        return row0;
    };
    switch (kind) {
        case VQB_CONV_K3: case VQB_CONVT_K3: case VQB_CONV_K1: {
            if (Cout % 16 != 0 || Cout < 16 || Cout > 256 || kc > HC_MAX_CHUNKS) return false;
            const int taps = kind == VQB_CONV_K1 ? 1 : 9;
            if (kc * taps > HC_MAX_STEPS) return false;
            pl.transposed = kind == VQB_CONVT_K3;
            pl.halo = kind == VQB_CONV_K1 ? 0 : 1;
            pl.nchunks = kc; pl.NCOL = Cout; pl.nbmax = Cout; pl.cg = Cout;
            for (int k = 0; k < kc; ++k) {
                pl.chunk_c0[k] = 64 * k; pl.chunk_p[k] = 0;
                for (int t = 0; t < taps; ++t) {
                    const int r = taps == 1 ? 0 : t / 3, s = taps == 1 ? 0 : t % 3;
                    const int dy = taps == 1 ? 0 : (pl.transposed ? 1 - r : r - 1), dx = taps == 1 ? 0 : (pl.transposed ? 1 - s : s - 1);
                    add_step(pl, 0, k, dy, dx, Cout, 0, rows_for(0, Cout, 64 * k, r, s), false);
                }
            }
            break;
        }
        case VQB_CONV_K4S2: {
            // encoder.py:32: out(y) reads in(2y + r - 1): r = 0 -> (Y = y-1, parity 1), 1 -> (y, 0), 2 -> (y, 1), 3 -> (y+1, 0)
            if (Cout % 16 != 0 || Cout < 16 || Cout > 256 || 4 * kc > HC_MAX_CHUNKS || 16 * kc > HC_MAX_STEPS) return false;
            pl.s2d = 1; pl.NCOL = Cout; pl.nbmax = Cout; pl.cg = Cout;
            static const int RR[2][2] = {{1, 3}, {0, 2}}, DD[2][2] = {{0, 1}, {-1, 0}};      // [parity][i] -> kernel row / shift
            for (int py = 0; py < 2; ++py)
                for (int px = 0; px < 2; ++px)
                    for (int k = 0; k < kc; ++k) {
                        const int ch = pl.nchunks++;
                        pl.chunk_c0[ch] = px * Cin + 64 * k; pl.chunk_p[ch] = py;
                        for (int a = 0; a < 2; ++a)
                            for (int b = 0; b < 2; ++b)
                                add_step(pl, 0, ch, DD[py][a], DD[px][b], Cout, 0, rows_for(0, Cout, 64 * k, RR[py][a], RR[px][b]), false);
                    }
            break;
        }
        case VQB_CONVT_K4S2: {
            // decoder.py:31: output row 2y+py takes input row y+dy through kernel row r = py + 1 - 2 dy:
            //   py = 0: (dy 0, r 1), (dy -1, r 3);  py = 1: (dy 0, r 2), (dy +1, r 0); same along x.
            if (Cout % 32 != 0 || Cout < 32 || 2 * Cout > 256 || kc > HC_MAX_CHUNKS || 6 * kc > HC_MAX_STEPS) return false;
            pl.transposed = 1; pl.npass = 2; pl.nchunks = kc; pl.NCOL = 2 * Cout; pl.nbmax = 2 * Cout; pl.nbhalf = Cout;
            pl.cg = Cout; pl.sy = 2; pl.sx = 2;
            static const int TR[2][2] = {{1, 3}, {2, 0}}, TD[2][2] = {{0, -1}, {0, 1}};
            for (int k = 0; k < kc; ++k) { pl.chunk_c0[k] = 64 * k; pl.chunk_p[k] = 0; }
            for (int py = 0; py < 2; ++py)
                for (int k = 0; k < kc; ++k)
                    for (int a = 0; a < 2; ++a) {
                        const int r = TR[py][a], dy = TD[py][a];
                        // dx = 0 feeds both column parities: [px 0 with s = 1 | px 1 with s = 2] -> one N = 2 Cout step
                        const int row0 = rows_for(0, Cout, 64 * k, r, 1);
                        rows_for(0, Cout, 64 * k, r, 2);
                        add_step(pl, py, k, dy, 0, 2 * Cout, 0, row0, false);
                        add_step(pl, py, k, dy, -1, Cout, 0, rows_for(0, Cout, 64 * k, r, 3), true);       // px 0, s = 3
                        add_step(pl, py, k, dy, 1, Cout, Cout, rows_for(0, Cout, 64 * k, r, 0), true);     // px 1, s = 0
                    }
            break;
        }
        case VQB_CONVT_K4S2_OUT: {
            // decoder.py:34: 16 columns (py, px, co); shift (dy,dx) reaches column (py,px,co) through r = py+1-2dy, s = px+1-2dx
            if (Cout < 1 || Cout > 4 || kc > HC_MAX_CHUNKS || 9 * kc > HC_MAX_STEPS) return false;
            pl.transposed = 1; pl.nchunks = kc; pl.NCOL = 16; pl.nbmax = 16; pl.cg = 16; pl.epi_mode = EPI_SHUFFLE_NCHW;
            for (int k = 0; k < kc; ++k) {
                pl.chunk_c0[k] = 64 * k; pl.chunk_p[k] = 0;
                for (int t = 0; t < 9; ++t) {
                    const int dy = t / 3 - 1, dx = t % 3 - 1;
                    const int row0 = (int)pl.rows.size();
                    for (int col = 0; col < 16; ++col) {
                        const int ph = col / Cout, co = col % Cout, py = ph >> 1, px = ph & 1;
                        const int r = py + 1 - 2 * dy, s = px + 1 - 2 * dx;
                        if (ph < 4 && r >= 0 && r <= 3 && s >= 0 && s <= 3) pl.rows.push_back({co, 64 * k, r, s});
                        else pl.rows.push_back({-1, 0, 0, 0});
                    }
                    add_step(pl, 0, k, dy, dx, 16, 0, row0, false);
                }
            }
            if (Cin == 64 && Cout == 3) {
                // the same layer in scatter form (convt_out_bf16.cu): 64 more rows, one per GEMM column (ky, kx, co)
                pl.scatter_row0 = (int)pl.rows.size();
                for (int n = 0; n < 64; ++n) {
                    int co, ky, kx;
                    convt_out_scatter_column(n, &co, &ky, &kx);
                    pl.rows.push_back({co, 0, ky, kx});
                }
            }
            break;
        }
        default: return false;
    }
    if (pl.rows.size() > 65535) return false;
    // flags: first write of each accumulator range, chunk boundaries
    for (int ps = 0; ps < pl.npass; ++ps) {
        bool seen[256] = {false};
        for (int i = 0; i < pl.nsteps[ps]; ++i) {
            PlanStep &s = pl.steps[ps][i];
            bool first = !seen[s.d_col];
            for (int c = s.d_col; c < s.d_col + s.nb; ++c) {
                if (first && seen[c]) return false;          // a partially written range cannot be overwritten
                if (!first && !seen[c]) return false;
            }
            if (first) { s.flags |= ST_FIRST; for (int c = s.d_col; c < s.d_col + s.nb; ++c) seen[c] = true; }
            if (i == 0 || pl.steps[ps][i - 1].chunk != s.chunk) s.flags |= ST_NEWCHUNK;
            if (i + 1 == pl.nsteps[ps] || pl.steps[ps][i + 1].chunk != s.chunk) s.flags |= ST_ENDCHUNK;
        }
    }
    return true;
}

const Plan *get_plan(int kind, int Cin, int Cout) {
    static std::vector<Plan *> cache;           // a handful of layer shapes per process; never freed
    for (Plan *pl : cache) if (pl->kind == kind && pl->Cin == Cin && pl->Cout == Cout) return pl;
    Plan *pl = new Plan();
    if (!build_plan(*pl, kind, Cin, Cout)) { delete pl; return nullptr; }
    cache.push_back(pl);
    return pl;
}

__global__ void hconv_pack_kernel(const float *__restrict__ w, const int4 *__restrict__ rows, int nrows, int Cout, int Cin,
                                  int kh, int kw, int transposed, __nv_bfloat16 *__restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nrows * 64) return;
    const int row = i >> 6, j = i & 63;
    const int4 d = rows[row];
    float v = 0.f;
    if (d.x >= 0 && d.y + j < Cin) {
        const int ci = d.y + j;
        v = transposed ? w[(((size_t)ci * Cout + d.x) * kh + d.z) * kw + d.w] : w[(((size_t)d.x * Cin + ci) * kh + d.z) * kw + d.w];
    }
    out[i] = __float2bfloat16_rn(v);
}


void kernel_dims(int kind, int &kh, int &kw) {
    kh = kw = (kind == VQB_CONV_K1 || kind == VQB_RES_W2_KIND) ? 1 : (kind == VQB_CONV_K3 || kind == VQB_CONVT_K3) ? 3 : 4;
}

}  // namespace

int hconv_plan_rows(int kind, int Cin, int Cout) {
    const Plan *pl = get_plan(kind, Cin, Cout);
    return pl ? (int)pl->rows.size() : -1;
}

extern "C" size_t vqb_conv_bf16_packed_bytes(int kind, int Cout, int Cin) {
    const Plan *pl = get_plan(kind, Cin, Cout);
    if (!pl) return 0;
    return pl->rows.size() * 128 + pl->rows.size() * sizeof(int4) + 256;
}

extern "C" int vqb_pack_conv_weight_bf16(const float *w, void *packed, int kind, int Cout, int Cin, void *stream) {
    if (!w || !packed) return VQB_ERR_BAD_ARG;
    const Plan *pl = get_plan(kind, Cin, Cout);
    if (!pl) return VQB_ERR_UNSUPPORTED;
    if (reinterpret_cast<uintptr_t>(packed) & 127) return VQB_ERR_ALIGNMENT;
    cudaStream_t s = (cudaStream_t)stream;
    const int nrows = (int)pl->rows.size();
    int4 *table = reinterpret_cast<int4 *>(reinterpret_cast<unsigned char *>(packed) + (size_t)nrows * 128);
    static_assert(sizeof(RowDesc) == sizeof(int4), "row table layout");
    cudaError_t e = cudaMemcpyAsync(table, pl->rows.data(), (size_t)nrows * sizeof(int4), cudaMemcpyHostToDevice, s);
    if (e != cudaSuccess) return (int)e;
    int kh, kw;
    kernel_dims(kind, kh, kw);
    hconv_pack_kernel<<<(nrows * 64 + 255) / 256, 256, 0, s>>>(w, table, nrows, Cout, Cin, kh, kw, pl->transposed,
                                                               reinterpret_cast<__nv_bfloat16 *>(packed));
    VQB_COUNT_LAUNCH(1);
    return vqb_cuda_status(cudaGetLastError());
}

namespace {

// first row of the block of Cout packed rows (co = 0 .. Cout-1) holding input channels [ci0, ci0 + 64) of tap (r, s)
int find_rows(const Plan &pl, int ci0, int r, int s) {
    const int n = (int)pl.rows.size();
    for (int i = 0; i + pl.Cout <= n; ++i) {
        const RowDesc &a = pl.rows[i], &b = pl.rows[i + pl.Cout - 1];
        if (a.co == 0 && a.ci0 == ci0 && a.r == r && a.s == s && b.co == pl.Cout - 1 && b.ci0 == ci0 && b.r == r && b.s == s)
            return i;
    }
    return -1;
}

}  // namespace

// in: bf16 NHWC (B, H, W, Cin).  out: bf16 NHWC (out_f32 = 0) / fp32 NHWC (out_f32 = 1) / fp32 NCHW (VQB_CONVT_K4S2_OUT).
extern "C" int vqb_conv2d_bf16(const void *in, const void *packed, const float *bias, void *out, int B, int Cin, int H, int W,
                               int Cout, int kind, int relu, int out_f32, void *stream) {
    if (!in || !packed || !out) return VQB_ERR_BAD_ARG;
    if (B <= 0 || Cin <= 0 || H <= 0 || W <= 0 || Cout <= 0) return VQB_ERR_BAD_ARG;
    const Plan *pl = get_plan(kind, Cin, Cout);
    if (!pl) return VQB_ERR_UNSUPPORTED;
    if ((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(packed)) & 15) return VQB_ERR_ALIGNMENT;
    if (pl->s2d && ((H | W) & 1)) return VQB_ERR_UNSUPPORTED;
    if (kind == VQB_CONVT_K4S2_OUT) out_f32 = 1;

    WgLaunch L;
    L.bf16 = 1;
    L.in = in; L.B = B; L.Cin = Cin; L.H = H; L.W = W; L.in_step = 1;
    L.w = packed; L.w_rows = (long long)pl->rows.size(); L.w_inner = 64;
    L.bias = bias; L.out = out; L.out_bf16 = !out_f32; L.relu = relu;
    L.ncols = Cout;
    // output: NHWC of the layer's output grid (strides in elements)
    const bool up = kind == VQB_CONVT_K4S2 || kind == VQB_CONVT_K4S2_OUT;
    const int OH = up ? 2 * H : pl->s2d ? H / 2 : H, OW = up ? 2 * W : pl->s2d ? W / 2 : W;
    L.out_sn = (long long)OH * OW * Cout; L.out_sh = (long long)OW * Cout; L.out_sw = Cout; L.out_sc = 1;
    L.nph = 1;
    L.OHg[0] = OH; L.OWg[0] = OW;
    const int kc = Cin / 64;
    auto add = [&](int ph, int c0, int dx, int dy, int row) {
        if (row < 0 || L.nsteps[ph] >= WG_MAX_STEPS) return false;
        L.steps[ph][L.nsteps[ph]++] = WgStep{c0, 0, dx, dy, row};
        return true;
    };
    switch (kind) {
        case VQB_CONV_K4S2:                 // out(y) reads in(2y + r - 1)
            L.in_step = 2;
            for (int r = 0; r < 4; ++r)
                for (int s = 0; s < 4; ++s)
                    for (int k = 0; k < kc; ++k)
                        if (!add(0, 64 * k, s - 1, r - 1, find_rows(*pl, 64 * k, r, s))) return VQB_ERR_UNSUPPORTED;
            break;
        case VQB_CONVT_K4S2:                // output (2y + py, 2x + px) takes input (y + dy, x + dx), kernel row r = py + 1 - 2 dy
            L.nph = 4; L.out_step = 2;
            for (int ph = 0; ph < 4; ++ph) {
                const int py = ph >> 1, px = ph & 1;
                L.OHg[ph] = H; L.OWg[ph] = W; L.out_py[ph] = py; L.out_px[ph] = px;
                for (int r = 0; r < 4; ++r) {
                    if ((py + 1 - r) % 2 != 0) continue;
                    for (int s = 0; s < 4; ++s) {
                        if ((px + 1 - s) % 2 != 0) continue;
                        for (int k = 0; k < kc; ++k)
                            if (!add(ph, 64 * k, (px + 1 - s) / 2, (py + 1 - r) / 2, find_rows(*pl, 64 * k, r, s))) return VQB_ERR_UNSUPPORTED;
                    }
                }
            }
            break;
        case VQB_CONVT_K4S2_OUT:            // N = 16 columns (sub-pixel phase, channel) per input pixel
            L.OHg[0] = H; L.OWg[0] = W; L.ncols = 4 * Cout; L.shuffle_cg = Cout;
            L.out_sn = (long long)Cout * OH * OW; L.out_sc = (long long)OH * OW; L.out_sh = OW; L.out_sw = 1;
            for (int i = 0; i < pl->nsteps[0]; ++i) {
                const PlanStep &st = pl->steps[0][i];
                if (!add(0, pl->chunk_c0[st.chunk], st.dx, st.dy, st.w_row)) return VQB_ERR_UNSUPPORTED;
            }
            break;
        default:                            // k1 / k3 convs and the k3 transposed conv: the plan's steps as they are
            for (int i = 0; i < pl->nsteps[0]; ++i) {
                const PlanStep &st = pl->steps[0][i];
                if (!add(0, pl->chunk_c0[st.chunk], st.dx, st.dy, st.w_row)) return VQB_ERR_UNSUPPORTED;
            }
            break;
    }
    L.N = wg_gemm_cols(L.ncols);
    if (L.N == 0) return VQB_ERR_UNSUPPORTED;
    return launch_wgconv(L, (cudaStream_t)stream);
}

bool res_bf16_supported(int C, int Cmid) {
    return (C == 64 || C == 128) && Cmid % 16 == 0 && Cmid >= 16 && Cmid <= 64;
}

// r, out: bf16 NHWC (B,H,W,C).  w1: packing of kind VQB_CONV_K3 with (Cout = Cmid, Cin = C); w2: VQB_RES_W2_KIND with
// (Cout = C, Cin = Cmid) -- both made by vqb_pack_conv_weight_bf16.  One launch: per 128-pixel tile the 3x3 GEMM, ReLU,
// and the 1x1 GEMM on the bf16 intermediate held in shared memory, + r, optional ReLU.
extern "C" int vqb_residual_layer_bf16(const void *r, const void *w1_packed, const void *w2_packed, void *out, int B, int H,
                                       int W, int C, int Cmid, int relu_out, void *stream) {
    if (!r || !w1_packed || !w2_packed || !out) return VQB_ERR_BAD_ARG;
    if (B <= 0 || H <= 0 || W <= 0 || C <= 0 || Cmid <= 0) return VQB_ERR_BAD_ARG;
    if (!res_bf16_supported(C, Cmid)) return VQB_ERR_UNSUPPORTED;
    if (r == out) return VQB_ERR_BAD_ARG;                       // neighbouring tiles read each other's halo: not in place
    if ((reinterpret_cast<uintptr_t>(r) | reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(w1_packed) |
         reinterpret_cast<uintptr_t>(w2_packed)) & 15) return VQB_ERR_ALIGNMENT;
    const Plan *p1 = get_plan(VQB_CONV_K3, C, Cmid), *p2 = get_plan(VQB_RES_W2_KIND, Cmid, C);
    if (!p1 || !p2) return VQB_ERR_UNSUPPORTED;
    WgLaunch L;
    L.bf16 = 1;
    L.in = r; L.B = B; L.Cin = C; L.H = H; L.W = W; L.in_step = 1;
    L.w = w1_packed; L.w_rows = (long long)p1->rows.size(); L.w_inner = 64;
    L.ncols = Cmid; L.N = wg_gemm_cols(Cmid);
    L.w2 = w2_packed; L.w2_rows = (long long)p2->rows.size(); L.N2 = C;
    L.skip = r; L.out = out; L.out_bf16 = 1; L.relu = relu_out;
    L.out_sn = (long long)H * W * C; L.out_sh = (long long)W * C; L.out_sw = C; L.out_sc = 1;
    L.nph = 1; L.OHg[0] = H; L.OWg[0] = W;
    for (int i = 0; i < p1->nsteps[0]; ++i) {
        const PlanStep &st = p1->steps[0][i];
        L.steps[0][i] = WgStep{p1->chunk_c0[st.chunk], 0, st.dx, st.dy, st.w_row};
    }
    L.nsteps[0] = p1->nsteps[0];
    return launch_wgconv(L, (cudaStream_t)stream);
}

// GEMM column n of the scatter form -> (co, ky, kx) of the ConvTranspose2d weight, or co = -1 for a padding column.
void convt_out_scatter_column(int n, int *co, int *ky, int *kx) {
    *co = -1; *ky = 0; *kx = 0;
    if (n < 12) { const int r = n / 6, s = (n / 3) & 1; *co = n % 3; *ky = r + 1; *kx = s + 1; return; }
    const int grp = (n - 12) / 8, j = (n - 12) % 8;
    if (n < 44) {
        if (j >= 6) return;
        const int a = j / 3;                     // s for the up / down groups, r for the left / right groups
        *co = j % 3;
        if (grp == 0) { *ky = 0; *kx = a + 1; }
        else if (grp == 1) { *ky = 3; *kx = a + 1; }
        else if (grp == 2) { *ky = a + 1; *kx = 0; }
        else { *ky = a + 1; *kx = 3; }
        return;
    }
    const int c = (n - 44) / 4, jj = (n - 44) % 4;
    if (c > 3 || jj >= 3) return;
    *co = jj; *ky = (c >> 1) ? 3 : 0; *kx = (c & 1) ? 3 : 0;
}

// (test hook, tests/test_abi_cpu.py: the column layout is host logic and is pinned without a GPU)
extern "C" int vqb_debug_convt_out_scatter_column(int n, int *co, int *ky, int *kx) {
    if (n < 0 || n >= 64 || !co || !ky || !kx) return VQB_ERR_BAD_ARG;
    convt_out_scatter_column(n, co, ky, kx);
    return 0;
}

