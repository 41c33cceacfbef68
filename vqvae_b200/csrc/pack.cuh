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
