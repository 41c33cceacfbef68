// pack.cuh -- the weight packings as index functions: element i of a packing, read from the parameter as PyTorch
// stores it.  The single-packing entry points (misc.cu, prior.cu) and the multi-packing launch (optim.cu) all write
// through these, so each layout has one definition.
#pragma once

// K-major rows [(r*kw+s)][co][ci] of Cin_pad >= Cin channels, zero padded, from a conv weight (Cout,Cin,kh,kw) or a
// transposed one (Cin,Cout,kh,kw): the B operand of every conv kernel.  i < kh*kw*Cout*Cin_pad.
__device__ __forceinline__ float pack_kmajor_at(const float *__restrict__ w, long long i, int Cout, int Cin,
                                                int Cin_pad, int kh, int kw, int transposed) {
    const int ci = (int)(i % Cin_pad);
    long long t = i / Cin_pad;
    const int co = (int)(t % Cout);
    const int tap = (int)(t / Cout);
    const int r = tap / kw, s = tap % kw;
    const long long src = transposed ? ((((long long)ci * Cout + co) * kh + r) * kw + s)
                                     : ((((long long)co * Cin + ci) * kh + r) * kw + s);
    return ci < Cin ? w[src] : 0.f;
}

// ConvTranspose2d k4 s2 p1 weight (Cin,Cout,4,4), Cout <= 4  ->  [9 neighbour taps (dy,dx)][16][Cin]: row
// (py*2+px)*Cout+co of tap (dy,dx) holds W[ci][co][py-2dy+1][px-2dx+1] when that kernel index exists (the neighbour
// contributes to that output phase), else 0.  Read by launch_convt_shuffle_wg (wgconv.cu).  i < 9*16*Cin.
__device__ __forceinline__ float pack_shuffle_at(const float *__restrict__ w, int i, int Cout, int Cin) {
    const int ci = i % Cin, row = (i / Cin) % 16, tap = i / (16 * Cin);
    const int dy = tap / 3 - 1, dx = tap % 3 - 1;
    float v = 0.f;
    if (row < 4 * Cout) {
        const int co = row % Cout, ph = row / Cout, py = ph >> 1, px = ph & 1;
        const int kh = py - 2 * dy + 1, kw = px - 2 * dx + 1;
        if (kh >= 0 && kh < 4 && kw >= 0 && kw < 4) v = w[(((size_t)ci * Cout + co) * 4 + kh) * 4 + kw];
    }
    return v;
}

// The prior's layout: conv weight (Cout, Cin, kh, kw) -> [(r*cols + s)*Cin + ci][co] for the kept taps r < rows,
// s < cols.  i < rows*cols*Cin*Cout.
__device__ __forceinline__ float pack_prior_at(const float *__restrict__ w, long long i, int Cout, int Cin, int kh,
                                               int kw, int cols) {
    const int co = (int)(i % Cout);
    const long long t = i / Cout;
    const int ci = (int)(t % Cin), tap = (int)(t / Cin);
    const int r = tap / cols, sc = tap % cols;
    return w[(((long long)co * Cin + ci) * kh + r) * kw + sc];
}

// The padded prior layouts (VQB_PACK_PRIOR_PAD_F32, _PAD_F32, _UNPAD_F32): a channel axis of n real channels and kind
// 0 (not padded), 1 (dim-wide: n -> cp) or 2 (a gate axis: 2*dim -> 2*cp, padded per half).
__host__ __device__ __forceinline__ int pad_width(int n, int kind, int cp) { return kind == 0 ? n : kind * cp; }

// real channel -> its padded index
__device__ __forceinline__ int pad_index(int c, int n, int kind, int cp) {
    if (kind == 0) return c;
    const int d = n / kind;
    return (c / d) * cp + c % d;
}

// padded index -> its real channel, or -1 for a padding channel
__device__ __forceinline__ int pad_real(int c, int n, int kind, int cp) {
    if (kind == 0) return c;
    const int d = n / kind, r = c % cp;
    return r < d ? (c / cp) * d + r : -1;
}

// VQB_PACK_PRIOR_PAD_F32: pack_prior_at of the zero-padded weight.  i < rows*cols*Cin'*Cout'.
__device__ __forceinline__ float pack_prior_pad_at(const float *__restrict__ w, long long i, int Cout, int Cin, int kh,
                                                   int kw, int cols, int cp, int kout, int kin) {
    const int coutp = pad_width(Cout, kout, cp), cinp = pad_width(Cin, kin, cp);
    const int co = pad_real((int)(i % coutp), Cout, kout, cp);
    const long long t = i / coutp;
    const int ci = pad_real((int)(t % cinp), Cin, kin, cp), tap = (int)(t / cinp);
    if (co < 0 || ci < 0) return 0.f;
    const int r = tap / cols, sc = tap % cols;
    return w[(((long long)co * Cin + ci) * kh + r) * kw + sc];
}

// VQB_PACK_PAD_F32: (Cout, Cin, khw) -> (Cout', Cin', khw), zero at the padding.  i < Cout'*Cin'*khw.
__device__ __forceinline__ float pack_pad_at(const float *__restrict__ w, long long i, int Cout, int Cin, int khw,
                                             int cp, int kout, int kin) {
    const int cinp = pad_width(Cin, kin, cp);
    const int tap = (int)(i % khw);
    const long long t = i / khw;
    const int ci = pad_real((int)(t % cinp), Cin, kin, cp), co = pad_real((int)(t / cinp), Cout, kout, cp);
    if (co < 0 || ci < 0) return 0.f;
    return w[((long long)co * Cin + ci) * khw + tap];
}

// VQB_PACK_UNPAD_F32: element i < Cout*Cin*khw of (Cout, Cin, khw), read from the padded (Cout', Cin', khw).
__device__ __forceinline__ float unpad_at(const float *__restrict__ w, long long i, int Cout, int Cin, int khw, int cp,
                                          int kout, int kin) {
    const int cinp = pad_width(Cin, kin, cp);
    const int tap = (int)(i % khw);
    const long long t = i / khw;
    const int ci = pad_index((int)(t % Cin), Cin, kin, cp), co = pad_index((int)(t / Cin), Cout, kout, cp);
    return w[((long long)co * cinp + ci) * khw + tap];
}
