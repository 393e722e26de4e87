// Standalone GPU check of the wgmma conv kernel against a plain CPU loop (bf16-rounded operands, double
// accumulation, the interval rule of oracle/conv_check.py).  Build: see __graft_entry__.build().  Run on an H100:
//   build/test_conv_tc [perf]   the bf16 / bf16x3 cases below (perf: then time the bench's layer shapes)
//   build/test_conv_tc matrix   every conv_tc_kernel instantiation at tile edges, exact-integer and interval operands,
//                               each case at seven grid sizes, bit for bit across them (run_matrix)
//   build/test_conv_tc list     the matrix's (format, N, ragged, PReLU) per case, without touching the GPU
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../pytorch_realtime_multi-person_pose_estimation_b200/csrc/conv_tc.cuh"
#include "../../pytorch_realtime_multi-person_pose_estimation_b200/csrc/f16_core.h"
#include "../../pytorch_realtime_multi-person_pose_estimation_b200/csrc/fp8_core.h"

using namespace b2p;

#define CK(x)                                                                          \
    do {                                                                               \
        cudaError_t e_ = (x);                                                          \
        if (e_ != cudaSuccess) {                                                       \
            printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); \
            exit(2);                                                                   \
        }                                                                              \
    } while (0)

static uint32_t rng_state = 12345;
static float frand() {
    rng_state = rng_state * 1664525u + 1013904223u;
    return ((rng_state >> 8) & 0xFFFF) / 65536.0f - 0.5f;
}
static float bf16r(float f) { return __bfloat162float(__float2bfloat16(f)); }

// round-to-nearest-even of a double to bf16 precision (one rounding) and the bf16 ulp of a bf16 value
static double bf16_rne(double d) {
    uint64_t u;
    memcpy(&u, &d, 8);
    u = (u + ((1ull << 44) - 1) + ((u >> 45) & 1)) & ~((1ull << 45) - 1);
    memcpy(&d, &u, 8);
    return d;
}
static double bf16_ulp(double v) {
    if (v == 0) return 0;
    int ex;
    std::frexp(v, &ex);
    return std::ldexp(1.0, ex - 8);
}

struct Case {
    const char* name;
    int n, H, W, ks, groups, cin_g, in_stride_g, cout_g, n_tile, relu, pool, head;
    int split;          // 1: run in bf16x3 only (hi + lo planes, three MMA terms, K-chunked); 0: see main
    int in_base, in_c;  // first input channel of group 0 / channels per input pixel (0: cin_g or cin_g * groups)
    int out_off, out_c; // first output channel of group 0 / channels per output pixel (0: groups * cout_g)
    int pdl;            // the input is written by a preceding launch (identity 1x1 conv) and this one is PDL-chained to it
};

// Every output is checked against the interval a correctly accumulated fp32 sum could round to (oracle/conv_check.py):
// r = sum(a * w) + b and S = sum|a * w| + |b| in double, e = 2^-22 * c * S with c from the kernel's accumulation
// structure, accept R(f(r - e)) <= got <= R(f(r + e)) (f = ReLU then 2x2 max, R = bf16 round-to-nearest-even).
// head: out_ch_off {0,40}, store {40,24}, f32 {38,19}; cout_g is the padded per-group Cout (n_tile).
static int run_case(const Case& c, int num_sms, TcFormat fmt) {
    const bool split = tc_planes(fmt) == 2;
    const char* fmt_name = split ? "bf16x3" : "bf16";
    const int taps = c.ks * c.ks, pad = c.ks / 2;
    const int cin_blocks = c.cin_g / 64;
    const int in_c = c.in_c ? c.in_c : ((c.in_stride_g == 0) ? c.cin_g : c.cin_g * c.groups);
    const int n_tiles = c.cout_g / c.n_tile;
    const int rows = c.groups * c.cout_g;
    const int Ho = c.pool ? c.H / 2 : c.H, Wo = c.pool ? c.W / 2 : c.W;
    const int out_c = c.head ? 64 : (c.out_c ? c.out_c : rows);
    const int nterms = split ? 3 : 1;

    // activations: hi = bf16(x) (lo = bf16(x - hi) in split mode); weights likewise
    std::vector<float> in((size_t)c.n * c.H * c.W * in_c), in_lo(in.size(), 0.f), w((size_t)taps * rows * c.cin_g),
        w_lo(w.size(), 0.f), bias(rows);
    for (size_t i = 0; i < in.size(); ++i) {
        const float x = frand();
        in[i] = bf16r(x);
        if (split) in_lo[i] = bf16r(x - in[i]);
    }
    const float ws = 1.0f / std::sqrt((float)(taps * c.cin_g));
    for (size_t i = 0; i < w.size(); ++i) {
        const float x = frand() * 2.f * ws * 1.7f;
        w[i] = bf16r(x);
        if (split) w_lo[i] = bf16r(x - w[i]);
    }
    for (auto& v : bias) v = frand() * 0.2f;
    const int valid[2] = {c.head ? 38 : c.cout_g, c.head ? 19 : c.cout_g};
    if (c.head)  // padded rows carry zero weights/bias, as the weight packer does
        for (int g = 0; g < c.groups; ++g)
            for (int r = valid[g]; r < c.cout_g; ++r) {
                bias[g * c.cout_g + r] = 0.f;
                for (int t = 0; t < taps; ++t)
                    for (int k = 0; k < c.cin_g; ++k)
                        w[((size_t)t * rows + g * c.cout_g + r) * c.cin_g + k] = w_lo[((size_t)t * rows + g * c.cout_g + r) * c.cin_g + k] = 0.f;
            }

    // the weight tensor map spans 2*taps slices: [hi taps | lo taps]
    std::vector<__nv_bfloat16> in_h(in.size()), in_lo_h(in.size()), w_h(2 * w.size());
    for (size_t i = 0; i < in.size(); ++i) { in_h[i] = __float2bfloat16(in[i]); in_lo_h[i] = __float2bfloat16(in_lo[i]); }
    for (size_t i = 0; i < w.size(); ++i) { w_h[i] = __float2bfloat16(w[i]); w_h[w.size() + i] = __float2bfloat16(w_lo[i]); }

    __nv_bfloat16 *d_in, *d_in_lo = nullptr, *d_w, *d_out, *d_out_lo = nullptr, *d_src = nullptr, *d_wid = nullptr;
    float *d_bias, *d_zero = nullptr, *d_f32[2] = {nullptr, nullptr};
    CK(cudaMalloc(&d_in, in_h.size() * 2));
    CK(cudaMalloc(&d_w, w_h.size() * 2));
    CK(cudaMalloc(&d_bias, bias.size() * 4));
    const size_t out_elems = (size_t)c.n * Ho * Wo * out_c;
    CK(cudaMalloc(&d_out, out_elems * 2));
    CK(cudaMemset(d_out, 0xFF, out_elems * 2));       // NaN: channels a launch must not touch keep this pattern
    if (c.pdl) {       // the producer copies d_src into d_in (still NaN when this launch starts)
        CK(cudaMalloc(&d_src, in_h.size() * 2));
        CK(cudaMemcpy(d_src, in_h.data(), in_h.size() * 2, cudaMemcpyHostToDevice));
        CK(cudaMemset(d_in, 0xFF, in_h.size() * 2));
    } else {
        CK(cudaMemcpy(d_in, in_h.data(), in_h.size() * 2, cudaMemcpyHostToDevice));
    }
    if (split) {
        CK(cudaMalloc(&d_in_lo, in_h.size() * 2));
        CK(cudaMalloc(&d_out_lo, out_elems * 2));
        CK(cudaMemcpy(d_in_lo, in_lo_h.data(), in_h.size() * 2, cudaMemcpyHostToDevice));
        CK(cudaMemset(d_out_lo, 0xFF, out_elems * 2));
    }
    CK(cudaMemcpy(d_w, w_h.data(), w_h.size() * 2, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_bias, bias.data(), bias.size() * 4, cudaMemcpyHostToDevice));
    if (c.head)
        for (int g = 0; g < 2; ++g) CK(cudaMalloc(&d_f32[g], (size_t)c.n * valid[g] * c.H * c.W * 4));

    ConvTcArgs a;
    memset(&a, 0, sizeof(a));
    a.n_img = c.n; a.H = c.H; a.W = c.W; a.ksize = c.ks; a.cin_blocks = cin_blocks;
    a.in_ch_base = c.in_base; a.in_ch_group_stride = c.in_stride_g; a.groups = c.groups;
    a.n_tile = c.n_tile; a.n_tiles = n_tiles; a.bias = d_bias; a.relu = c.relu; a.pool = c.pool;
    a.out = d_out; a.out_cstride = out_c;
    for (int g = 0; g < 2; ++g) {
        a.out_ch_off[g] = c.head ? (g == 0 ? 0 : 40) : c.out_off + g * c.cout_g;
        a.store_ch[g] = c.head ? (g == 0 ? 40 : 24) : c.n_tile;
        a.out_f32[g] = d_f32[g];
        a.f32_ch[g] = c.head ? valid[g] : 0;
    }
    a.fmt = fmt;
    a.out_lo = d_out_lo;
    a.pdl = c.pdl;
    CK(conv_tc_make_maps(a, d_in, in_c, d_w, d_in_lo));
    if (c.pdl) {       // producer: 1x1 identity conv d_src -> d_in (exact: one product 1 * x per output)
        std::vector<__nv_bfloat16> wid((size_t)2 * in_c * in_c, __float2bfloat16(0.f));
        for (int o = 0; o < in_c; ++o) wid[(size_t)o * in_c + o] = __float2bfloat16(1.f);
        CK(cudaMalloc(&d_wid, wid.size() * 2));
        CK(cudaMalloc(&d_zero, in_c * 4));
        CK(cudaMemcpy(d_wid, wid.data(), wid.size() * 2, cudaMemcpyHostToDevice));
        CK(cudaMemset(d_zero, 0, in_c * 4));
        ConvTcArgs p;
        memset(&p, 0, sizeof(p));
        p.n_img = c.n; p.H = c.H; p.W = c.W; p.ksize = 1; p.cin_blocks = in_c / 64; p.groups = 1;
        p.n_tile = 64; p.n_tiles = in_c / 64; p.bias = d_zero; p.out = d_in; p.out_cstride = in_c; p.store_ch[0] = 64;
        CK(conv_tc_make_maps(p, d_src, in_c, d_wid));
        CK(conv_tc_launch(p, num_sms, 0));
    }
    CK(conv_tc_launch(a, num_sms, 0));
    cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) {
        printf("case %-34s %-6s : KERNEL FAILED: %s\n", c.name, fmt_name, cudaGetErrorString(e));
        return 100;
    }
#ifdef B2P_CONV_TIMELINE
    {
        std::vector<unsigned long long> tl(64 * kTlSlots);
        CK(conv_tc_read_timeline(tl.data()));
        const char* names[10] = {"entry", "prologue done", "patch cb0", "patch cb1", "first weights", "MMAs issued", "acc complete",
                                 "tile stored", "before final sync", "exit"};
        for (int cta = 0; cta < 4; ++cta) {
            printf("  timeline %s %s CTA %d (clk since entry):", c.name, fmt_name, cta);
            for (int sl = 1; sl < 10; ++sl) {
                const unsigned long long v = tl[cta * kTlSlots + sl], v0 = tl[cta * kTlSlots];
                printf(" %s=%lld", names[sl], v ? (long long)(v - v0) : -1LL);
            }
            printf("\n");
        }
    }
#endif
    std::vector<__nv_bfloat16> out_h(out_elems), out_lo_h(split ? out_elems : 0);
    CK(cudaMemcpy(out_h.data(), d_out, out_elems * 2, cudaMemcpyDeviceToHost));
    if (split) CK(cudaMemcpy(out_lo_h.data(), d_out_lo, out_elems * 2, cudaMemcpyDeviceToHost));
    std::vector<float> f32_h[2];
    if (c.head)
        for (int g = 0; g < 2; ++g) {
            f32_h[g].resize((size_t)c.n * valid[g] * c.H * c.W);
            CK(cudaMemcpy(f32_h[g].data(), d_f32[g], f32_h[g].size() * 4, cudaMemcpyDeviceToHost));
        }

    // CPU reference: r and S per pre-pool output, in double
    std::vector<double> ref((size_t)c.n * c.H * c.W * rows), sabs(ref.size());
    for (int n = 0; n < c.n; ++n)
        for (int y = 0; y < c.H; ++y)
            for (int x = 0; x < c.W; ++x)
                for (int g = 0; g < c.groups; ++g)
                    for (int co = 0; co < c.cout_g; ++co) {
                        double acc = bias[g * c.cout_g + co], sa = std::fabs(bias[g * c.cout_g + co]);
                        for (int dy = 0; dy < c.ks; ++dy) {
                            int yy = y + dy - pad;
                            if (yy < 0 || yy >= c.H) continue;
                            for (int dx = 0; dx < c.ks; ++dx) {
                                int xx = x + dx - pad;
                                if (xx < 0 || xx >= c.W) continue;
                                const size_t ib = ((size_t)(n * c.H + yy) * c.W + xx) * in_c + c.in_base + g * c.in_stride_g;
                                const size_t wb = ((size_t)(dy * c.ks + dx) * rows + g * c.cout_g + co) * c.cin_g;
                                for (int k = 0; k < c.cin_g; ++k) {
                                    const double ah = in[ib + k], al = in_lo[ib + k], wh = w[wb + k], wl = w_lo[wb + k];
                                    acc += ah * wh;
                                    sa += std::fabs(ah * wh);
                                    if (split) {      // A_hi W_lo + A_lo W_hi
                                        acc += ah * wl + al * wh;
                                        sa += std::fabs(ah * wl) + std::fabs(al * wh);
                                    }
                                }
                            }
                        }
                        ref[((size_t)(n * c.H + y) * c.W + x) * rows + g * c.cout_g + co] = acc;
                        sabs[((size_t)(n * c.H + y) * c.W + x) * rows + g * c.cout_g + co] = sa;
                    }
    // e = 2^-22 * coef * S (oracle/conv_check.py bound_coef)
    double coef;
    if (tc_chunked(fmt)) coef = c.ks == 7 ? 28 + 16 + nterms * cin_blocks * 7 : taps * 4 + 16 + nterms * cin_blocks;
    else coef = std::ceil(nterms * taps * c.cin_g / 16.0) + 16;
    const double U = std::ldexp(1.0, -22);
    auto fpos = [&](double v) { return c.relu && v < 0 ? 0.0 : v; };
    double max_ratio = 0, max_ratio32 = 0;
    long bad = 0, checked = 0;
    int printed = 0;
    for (int n = 0; n < c.n; ++n)
        for (int yo = 0; yo < Ho; ++yo)
            for (int xo = 0; xo < Wo; ++xo) {
                std::vector<bool> mine(out_c, false);
                for (int g = 0; g < c.groups; ++g) {
                    const int nstore = c.head ? (g == 0 ? 40 : 24) : c.cout_g;
                    for (int co = 0; co < nstore; ++co) {
                        const size_t col = (size_t)g * c.cout_g + co;
                        double flo = -1e300, fhi = -1e300, fr = -1e300, ef = 0;
                        for (int j = 0; j < (c.pool ? 4 : 1); ++j) {
                            const int y = c.pool ? 2 * yo + (j >> 1) : yo, x = c.pool ? 2 * xo + (j & 1) : xo;
                            const size_t ri = ((size_t)(n * c.H + y) * c.W + x) * rows + col;
                            const double e = U * coef * sabs[ri];
                            flo = std::max(flo, fpos(ref[ri] - e));
                            fhi = std::max(fhi, fpos(ref[ri] + e));
                            fr = std::max(fr, fpos(ref[ri]));
                            ef = std::max(ef, e);
                        }
                        const int oc = (c.head ? (g == 0 ? 0 : 40) : c.out_off + g * c.cout_g) + co;
                        mine[oc] = true;
                        const size_t oi = ((size_t)(n * Ho + yo) * Wo + xo) * out_c + oc;
                        const double got = __bfloat162float(out_h[oi]);
                        bool ok;
                        double dist;
                        if (split) {
                            const double lo = __bfloat162float(out_lo_h[oi]), wsl = std::ldexp(std::fabs(fr), -16);
                            ok = got + lo >= flo - wsl && got + lo <= fhi + wsl && std::fabs(lo) <= bf16_ulp(got) / 2;
                            dist = std::max(0.0, std::fabs(got + lo - fr) - wsl);
                        } else {
                            ok = got >= bf16_rne(flo) && got <= bf16_rne(fhi);
                            dist = std::max(0.0, std::fabs(got - fr) - bf16_ulp(got) / 2);
                        }
                        if (c.head && co >= valid[g]) ok = got == 0 && (!split || __bfloat162float(out_lo_h[oi]) == 0);
                        ++checked;
                        if (ef > 0) max_ratio = std::max(max_ratio, dist / ef);
                        if (!ok) {
                            if (printed++ < 5)
                                printf("  bad: n=%d y=%d x=%d ch=%d got %.9g interval [%.9g, %.9g]\n", n, yo, xo, oc, got,
                                       split ? flo : bf16_rne(flo), split ? fhi : bf16_rne(fhi));
                            ++bad;
                        }
                        if (c.head && co < valid[g]) {
                            const size_t ri = ((size_t)(n * c.H + yo) * c.W + xo) * rows + col;
                            const double e = U * coef * sabs[ri];
                            const double g32 = f32_h[g][((size_t)(n * valid[g] + co) * c.H + yo) * c.W + xo];
                            const double e32 = std::fabs(g32 - ref[ri]);
                            if (!(e32 <= e)) ++bad;
                            if (e > 0) max_ratio32 = std::max(max_ratio32, e32 / e);
                        }
                    }
                }
                // channels outside the launch's slice keep the fill pattern
                for (int oc = 0; oc < out_c; ++oc) {
                    if (mine[oc]) continue;
                    const size_t oi = ((size_t)(n * Ho + yo) * Wo + xo) * out_c + oc;
                    uint16_t bits, lbits = 0xFFFF;
                    memcpy(&bits, &out_h[oi], 2);
                    if (split) memcpy(&lbits, &out_lo_h[oi], 2);
                    if (bits != 0xFFFF || lbits != 0xFFFF) ++bad;
                }
            }
    printf("case %-34s %-6s : %ld outputs, max|v-r|/e bf16 %.3f f32 %.3f  bad=%ld  %s\n", c.name, fmt_name, checked,
           max_ratio, max_ratio32, bad, bad == 0 ? "OK" : "MISMATCH");
    cudaFree(d_in); cudaFree(d_w); cudaFree(d_bias); cudaFree(d_out);
    if (d_in_lo) cudaFree(d_in_lo);
    if (d_out_lo) cudaFree(d_out_lo);
    if (d_src) cudaFree(d_src);
    if (d_wid) cudaFree(d_wid);
    if (d_zero) cudaFree(d_zero);
    for (int g = 0; g < 2; ++g) if (d_f32[g]) cudaFree(d_f32[g]);
    return bad == 0 ? 0 : 1;
}

static void perf(int num_sms) {
    // Mconv{2..5}_stageX_L{1,2}: 7x7 128->128, both branches grouped, batch 32 @46x46.
    struct P { const char* name; int n, H, W, ks, groups, cin_g, stride_g, cout_g, n_tile, pool; };
    const P ps[] = {
        {"7x7 128->128 x2br b32 46^2", 32, 46, 46, 7, 2, 128, 128, 128, 128, 0},
        {"7x7 192->128 x2br b32 46^2", 32, 46, 46, 7, 2, 192, 0, 128, 128, 0},
        {"3x3 64->64 +pool b32 368^2", 32, 368, 368, 3, 1, 64, 64, 64, 64, 1},
        {"3x3 128->128 +pool b32 184^2", 32, 184, 184, 3, 1, 128, 128, 128, 128, 1},
        {"3x3 256->256 b32 92^2", 32, 92, 92, 3, 1, 256, 256, 256, 128, 0},
        {"3x3 512->512 b32 46^2", 32, 46, 46, 3, 1, 512, 512, 512, 128, 0},
        {"7x7 128->128 x2br b1 46^2", 1, 46, 46, 7, 2, 128, 128, 128, 128, 0},
    };
    for (const P& p : ps) {
        const int taps = p.ks * p.ks;
        const int in_c = p.stride_g == 0 ? p.cin_g : p.cin_g * p.groups;
        const int rows = p.groups * p.cout_g;
        const int Ho = p.pool ? p.H / 2 : p.H, Wo = p.pool ? p.W / 2 : p.W;
        __nv_bfloat16 *d_in, *d_w, *d_out;
        float* d_bias;
        size_t in_b = (size_t)p.n * p.H * p.W * in_c * 2, w_b = (size_t)2 * taps * rows * p.cin_g * 2;
        size_t out_b = (size_t)p.n * Ho * Wo * rows * 2;
        CK(cudaMalloc(&d_in, in_b)); CK(cudaMalloc(&d_w, w_b)); CK(cudaMalloc(&d_out, out_b));
        CK(cudaMalloc(&d_bias, rows * 4));
        CK(cudaMemset(d_in, 0x3c, in_b)); CK(cudaMemset(d_w, 0x3c, w_b)); CK(cudaMemset(d_bias, 0, rows * 4));
        ConvTcArgs a;
        memset(&a, 0, sizeof(a));
        a.n_img = p.n; a.H = p.H; a.W = p.W; a.ksize = p.ks; a.cin_blocks = p.cin_g / 64;
        a.in_ch_group_stride = p.stride_g; a.groups = p.groups; a.n_tile = p.n_tile; a.n_tiles = p.cout_g / p.n_tile;
        a.bias = d_bias; a.relu = 1; a.pool = p.pool; a.out = d_out; a.out_cstride = rows;
        for (int g = 0; g < 2; ++g) { a.out_ch_off[g] = g * p.cout_g; a.store_ch[g] = p.n_tile; }
        CK(conv_tc_make_maps(a, d_in, in_c, d_w));
        cudaEvent_t e0, e1;
        cudaEventCreate(&e0); cudaEventCreate(&e1);
        for (int i = 0; i < 3; ++i) CK(conv_tc_launch(a, num_sms, 0));
        CK(cudaDeviceSynchronize());
        const int iters = 10;
        cudaEventRecord(e0);
        for (int i = 0; i < iters; ++i) CK(conv_tc_launch(a, num_sms, 0));
        cudaEventRecord(e1);
        CK(cudaDeviceSynchronize());
        float ms;
        cudaEventElapsedTime(&ms, e0, e1);
        ms /= iters;
        double flops = 2.0 * p.n * p.H * p.W * (double)rows * taps * p.cin_g;
        printf("perf %-30s : %8.3f ms  %8.1f TFLOP/s\n", p.name, ms, flops / ms * 1e-9);
        cudaFree(d_in); cudaFree(d_w); cudaFree(d_out); cudaFree(d_bias);
    }
}

// ================================================ matrix ================================================
// One or more cases per conv_tc_kernel<F, N, kRagged, kPrelu> instantiation, at partial tiles (every residue of W mod 8
// and H mod 16), images down to 1x1 under 7x7 taps, 1 / 3 / >= 4 channel blocks, shared and strided groups, several
// n-tiles, pooling to odd extents, channel slices, the stage heads and ragged extents.  Each case runs in two operand
// modes:
//   exact   operands in {-1, 0, 1} (times a power of two per image for fp8's scales and fp16's overflow image),
//           bf16x3 residuals +-2^-9, integer or power-of-two biases and PReLU slopes {0.25, -0.5, 0, 1}.  Every
//           term is a multiple of the case's quantum q, the largest term M is at most 2^12 q and every output has
//           S = sum|a w| + |b| <= 2^12 M (asserted before the launch), so every partial sum in any order is exact in
//           fp32; fp8's k32 steps only add equal-magnitude terms of one (image, row), which its 13-bit accumulator
//           (DESIGN.md §3) also holds exactly.  Every stored word, residual word, fp32 map element and the amax, ea
//           and overflow tables are then known exactly and compared bit for bit.
//   random  the interval rule of run_case (bf16, bf16x3), with binary16 rounding for fp16 (tests/fp16_check.py) and
//           the min / max rule of tests/prelu_check.py for PReLU.  Not for fp8 (tests/test_gpu_fp8.py).
// Each case runs at the grid sizes 1, 2, 3, 7, S - 1, S and 2 S (S = SM count; the launch clamps to the tile count): the
// run at S is checked against the reference, every other run must equal it bit for bit, since each tile has one fixed
// MMA order and the fp8 amax and fp16 overflow updates do not depend on order.  Output buffers start as NaN (channels
// outside the launch's slice must keep it) and every output, fp32 map and per-image table sits between 4 KB sentinels.
namespace mx {

struct MCase {
    const char* name;
    TcFormat fmt;
    int N, ragged, prelu;
    int n, H, W, ks, groups, cin_g, in_stride_g, cout_g, relu, pool, head;
    int in_base, in_c, out_off, out_c;   // as in Case (0: the default)
    int ext_shift;   // ragged: log2 of the network input size over the launch's output size
    int ovf;         // fp16, exact mode: image 1's activations are 2^12, so that its outputs overflow binary16
};

const char* fmt_name(TcFormat f) {
    return f == TcFormat::kBf16 ? "bf16" : f == TcFormat::kBf16x3 ? "bf16x3" : f == TcFormat::kFp8 ? "fp8" : "fp16";
}

constexpr TcFormat B = TcFormat::kBf16, X3 = TcFormat::kBf16x3, F8 = TcFormat::kFp8, F16 = TcFormat::kFp16;
// clang-format off
const MCase kCases[] = {
    // name                            fmt  N  rag pr  n   H   W ks g cin strd cout relu pool head  base in_c off out_c shift ovf
    {"3x3 64->256 nt128x2",            B, 128, 0, 0,   3, 20, 13, 3, 1,  64,  0, 256, 1, 0, 0,    0,   0,  0,   0, 0, 0},
    {"3x3 192->128 pool cb3",          B, 128, 1, 0,   3, 36, 22, 3, 1, 192,  0, 128, 1, 1, 0,    0,   0,  0,   0, 1, 0},
    {"7x7 2grp 128->128 1x1 images",   B,  64, 0, 0,   3,  1,  1, 7, 2, 128,128, 128, 1, 0, 0,    0,   0,  0,   0, 0, 0},
    {"1x1 256->128 cb4",               B,  64, 1, 0,   4, 17,  9, 1, 1, 256,  0, 128, 1, 0, 0,    0,   0,  0,   0, 0, 0},
    {"1x1 head 128->38|19",            B,  48, 0, 0,   3, 15,  7, 1, 2, 128,128,  48, 0, 0, 1,    0,   0,  0,   0, 0, 0},
    {"7x7 head shared 128->38|19",     B,  48, 1, 0,   3, 18, 10, 7, 2, 128,  0,  48, 0, 0, 1,    0,   0,  0,   0, 0, 0},
    {"3x3 in 64..191/192 pool -> 64..191/192", B, 32, 0, 0, 3, 14, 12, 3, 1, 128, 0, 128, 1, 1, 0, 64, 192, 64, 192, 0, 0},
    {"7x7 2grp 128->64 nt32x2",        B,  32, 1, 0,   3, 21, 19, 7, 2, 128,128,  64, 1, 0, 0,    0,   0,  0,   0, 3, 0},
    {"3x3 128->128 prelu",             B, 128, 0, 1,   3, 23,  8, 3, 1, 128,  0, 128, 0, 0, 0,    0,   0,  0,   0, 0, 0},
    {"1x1 192->256 prelu cb3",         B, 128, 1, 1,   3, 13, 11, 1, 1, 192,  0, 256, 0, 0, 0,    0,   0,  0,   0, 0, 0},
    {"7x7 2grp shared 64->64 prelu",   B,  64, 0, 1,   3,  9,  6, 7, 2,  64,  0,  64, 0, 0, 0,    0,   0,  0,   0, 0, 0},
    {"3x3 64->128 prelu nt64x2",       B,  64, 1, 1,   4, 30, 20, 3, 1,  64,  0, 128, 0, 0, 0,    0,   0,  0,   0, 0, 0},
    {"1x1 64->96 prelu nt48x2",        B,  48, 0, 1,   3, 11,  5, 1, 1,  64,  0,  96, 0, 0, 0,    0,   0,  0,   0, 0, 0},
    {"3x3 128->48 prelu",              B,  48, 1, 1,   3, 25, 17, 3, 1, 128,  0,  48, 0, 0, 0,    0,   0,  0,   0, 0, 0},
    {"3x3 192->64 prelu nt32x2",       B,  32, 0, 1,   3, 12,  2, 3, 1, 192,  0,  64, 0, 0, 0,    0,   0,  0,   0, 0, 0},
    {"7x7 64->32 prelu",               B,  32, 1, 1,   3, 27, 15, 7, 1,  64,  0,  32, 0, 0, 0,    0,   0,  0,   0, 0, 0},
    {"7x7 2grp 128->64",              X3,  64, 0, 0,   3, 10,  7, 7, 2, 128,128,  64, 1, 0, 0,    0,   0,  0,   0, 0, 0},
    {"3x3 64->128 pool nt64x2",       X3,  64, 1, 0,   3, 34, 20, 3, 1,  64,  0, 128, 1, 1, 0,    0,   0,  0,   0, 2, 0},
    {"1x1 head 128->38|19",           X3,  48, 0, 0,   3,  7,  3, 1, 2, 128,128,  48, 0, 0, 1,    0,   0,  0,   0, 0, 0},
    {"7x7 head 128->38|19",           X3,  48, 1, 0,   3, 16, 12, 7, 2, 128,128,  48, 0, 0, 1,    0,   0,  0,   0, 0, 0},
    {"1x1 in 64..319/320 cb4 nt32x2", X3,  32, 0, 0,   3, 19, 14, 1, 1, 256,  0,  64, 1, 0, 0,   64, 320,  0,   0, 0, 0},
    {"3x3 64->32",                    X3,  32, 1, 0,   3,  6,  5, 3, 1,  64,  0,  32, 1, 0, 0,    0,   0,  0,   0, 0, 0},
    {"3x3 128->64 prelu",             X3,  64, 0, 1,   3, 17, 10, 3, 1, 128,  0,  64, 0, 0, 0,    0,   0,  0,   0, 0, 0},
    {"7x7 2grp shared 64->64 prelu",  X3,  64, 1, 1,   3,  8,  8, 7, 2,  64,  0,  64, 0, 0, 0,    0,   0,  0,   0, 0, 0},
    {"3x3 192->48 prelu cb3",         X3,  48, 0, 1,   3,  5,  9, 3, 1, 192,  0,  48, 0, 0, 0,    0,   0,  0,   0, 0, 0},
    {"1x1 64->96 prelu nt48x2",       X3,  48, 1, 1,   3, 31, 13, 1, 1,  64,  0,  96, 0, 0, 0,    0,   0,  0,   0, 2, 0},
    {"7x7 128->32 prelu 1x1 images",  X3,  32, 0, 1,   3,  1,  1, 7, 1, 128,  0,  32, 0, 0, 0,    0,   0,  0,   0, 0, 0},
    {"3x3 256->64 prelu cb4 nt32x2",  X3,  32, 1, 1,   3, 13, 22, 3, 1, 256,  0,  64, 0, 0, 0,    0,   0,  0,   0, 0, 0},
    {"3x3 128->128 pool nt64x2",      F8,  64, 0, 0,   3, 22, 18, 3, 1, 128,  0, 128, 1, 1, 0,    0,   0,  0,   0, 0, 0},
    {"7x7 2grp 128->64",              F8,  64, 1, 0,   3, 12, 11, 7, 2, 128,128,  64, 1, 0, 0,    0,   0,  0,   0, 0, 0},
    {"1x1 head 128->38|19",           F8,  48, 0, 0,   3, 20, 21, 1, 2, 128,128,  48, 0, 0, 1,    0,   0,  0,   0, 0, 0},
    {"7x7 head 128->38|19",           F8,  48, 1, 0,   3,  3,  4, 7, 2, 128,128,  48, 0, 0, 1,    0,   0,  0,   0, 0, 0},
    {"1x1 in 64..255/256 cb3 -> 32..95/128", F8, 32, 0, 0, 3, 9, 26, 1, 1, 192, 0, 64, 1, 0, 0,  64, 256, 32, 128, 0, 0},
    {"3x3 64->32 pool",               F8,  32, 1, 0,   4, 14, 10, 3, 1,  64,  0,  32, 1, 1, 0,    0,   0,  0,   0, 1, 0},
    {"3x3 64->128",                  F16, 128, 0, 0,   3, 29, 13, 3, 1,  64,  0, 128, 1, 0, 0,    0,   0,  0,   0, 0, 0},
    {"1x1 128->256 pool nt128x2",    F16, 128, 1, 0,   3, 26, 14, 1, 1, 128,  0, 256, 1, 1, 0,    0,   0,  0,   0, 1, 0},
    {"7x7 2grp 128->64 2x2 images",  F16,  64, 0, 0,   3,  2,  2, 7, 2, 128,128,  64, 1, 0, 0,    0,   0,  0,   0, 0, 0},
    {"3x3 192->64 cb3",              F16,  64, 1, 0,   3, 24, 23, 3, 1, 192,  0,  64, 1, 0, 0,    0,   0,  0,   0, 0, 0},
    {"1x1 head 128->38|19",          F16,  48, 0, 0,   3, 10,  9, 1, 2, 128,128,  48, 0, 0, 1,    0,   0,  0,   0, 0, 0},
    {"7x7 head shared 128->38|19",   F16,  48, 1, 0,   3, 17,  6, 7, 2, 128,  0,  48, 0, 0, 1,    0,   0,  0,   0, 0, 0},
    {"3x3 in 0..255/384 cb4 nt32x2", F16,  32, 0, 0,   3,  4, 15, 3, 1, 256,  0,  64, 1, 0, 0,    0, 384,  0,   0, 0, 0},
    {"1x1 64->32 5 images",          F16,  32, 1, 0,   5, 33,  9, 1, 1,  64,  0,  32, 1, 0, 0,    0,   0,  0,   0, 0, 0},
    {"3x3 64->128 image 1 overflows",F16, 128, 0, 0,   3, 16,  8, 3, 1,  64,  0, 128, 0, 0, 0,    0,   0,  0,   0, 0, 1},
    // more tiles than 2 S: at S - 1, S and 2 S the CTAs run 2 to 3 tiles each, across images
    {"1x1 64->256 nt128x2 persistent", B, 128, 0, 0,   4, 78, 70, 1, 1,  64,  0, 256, 1, 0, 0,    0,   0,  0,   0, 0, 0},
    {"1x1 64->64 prelu persistent",    B,  32, 1, 1,   3, 80, 72, 1, 1,  64,  0,  64, 0, 0, 0,    0,   0,  0,   0, 0, 0},
    {"1x1 64->64 nt32x2 persistent",  X3,  32, 1, 0,   4, 64, 72, 1, 1,  64,  0,  64, 1, 0, 0,    0,   0,  0,   0, 0, 0},
    {"1x1 64->128 nt64x2 persistent", F8,  64, 0, 0,   4, 80, 70, 1, 1,  64,  0, 128, 1, 0, 0,    0,   0,  0,   0, 0, 0},
    {"1x1 64->128 pool persistent",  F16,  64, 0, 0,   3, 96, 64, 1, 1,  64,  0, 128, 1, 1, 0,    0,   0,  0,   0, 0, 0},
};
// clang-format on

// ---- host rounding (one rounding from double) and bit patterns
double f16_rne(double d) {
    const double a = std::fabs(d);
    if (a >= 65520.0) return std::copysign(INFINITY, d);
    if (a < std::ldexp(1.0, -14)) return std::nearbyint(d * 16777216.0) / 16777216.0;   // subnormal step 2^-24, ties to even
    uint64_t u;
    memcpy(&u, &d, 8);
    u = (u + ((1ull << 41) - 1) + ((u >> 42) & 1)) & ~((1ull << 42) - 1);
    memcpy(&d, &u, 8);
    return d;
}
double f16_ulp(double v) {
    if (std::fabs(v) < std::ldexp(1.0, -14)) return std::ldexp(1.0, -24);
    int ex;
    std::frexp(v, &ex);
    return std::ldexp(1.0, ex - 11);
}
uint16_t bf16_bits(double v) {   // v: a bf16 value (or +-inf)
    const float f = (float)v;
    uint32_t u;
    memcpy(&u, &f, 4);
    return (uint16_t)(u >> 16);
}
double bf16_val(uint16_t b) {
    const uint32_t u = (uint32_t)b << 16;
    float f;
    memcpy(&f, &u, 4);
    return f;
}
double f16_val(uint16_t b) {
    const int s = b >> 15, e = (b >> 10) & 31, m = b & 1023;
    const double v = e == 31 ? (m ? NAN : INFINITY) : e == 0 ? std::ldexp((double)m, -24) : std::ldexp(1024.0 + m, e - 25);
    return s ? -v : v;
}
uint32_t f32_bits(float f) {
    uint32_t u;
    memcpy(&u, &f, 4);
    return u;
}
double r32(double v) { return (double)(float)v; }

// ---- device buffers between sentinels
constexpr size_t kGuard = 4096;
constexpr uint8_t kSentinel = 0x5A;
struct GBuf {
    uint8_t* base = nullptr;
    size_t bytes = 0, alloc = 0;
    void* p() const { return base ? base + kGuard : nullptr; }
};
GBuf galloc(size_t bytes) {
    GBuf g;
    g.bytes = bytes;
    g.alloc = kGuard + (bytes + 255) / 256 * 256 + kGuard;
    CK(cudaMalloc(&g.base, g.alloc));
    return g;
}
void gfill(const GBuf& g, int fill) {
    if (!g.base) return;
    CK(cudaMemset(g.base, kSentinel, g.alloc));
    CK(cudaMemset(g.base + kGuard, fill, g.bytes));
}
std::vector<uint8_t> gread(const GBuf& g) {
    std::vector<uint8_t> h(g.alloc);
    if (g.base) CK(cudaMemcpy(h.data(), g.base, g.alloc, cudaMemcpyDeviceToHost));
    return h;
}
long guard_damage(const std::vector<uint8_t>& h, const GBuf& g) {
    long bad = 0;
    for (size_t i = 0; i < h.size(); ++i)
        if ((i < kGuard || i >= kGuard + g.bytes) && h[i] != kSentinel) ++bad;
    return bad;
}
template <class T> T* upload(const std::vector<T>& v) {
    T* d = nullptr;
    CK(cudaMalloc(&d, v.size() * sizeof(T) + 16));
    CK(cudaMemcpy(d, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
    return d;
}

// worst |v - r| / e per (format, N, ragged, PReLU), random mode: 16-bit words and fp32 maps
struct Worst {
    double w16 = 0, w32 = 0;
    bool seen = false;
};
Worst g_worst[4][129][2][2];

// One case in one operand mode at every grid size.  Returns 0, 1 (mismatch) or 100 (kernel failure).
int run(const MCase& c, int ci, bool exact, int sms) {
    const TcFormat F = c.fmt;
    const bool split = F == X3, fp8 = F == F8, f16 = F == F16;
    const int taps = c.ks * c.ks, pad = c.ks / 2, cb = c.cin_g / 64;
    const int in_c = c.in_c ? c.in_c : (c.in_stride_g == 0 ? c.cin_g : c.cin_g * c.groups);
    const int n_tiles = c.cout_g / c.N, rows = c.groups * c.cout_g;
    const int Ho = c.pool ? c.H / 2 : c.H, Wo = c.pool ? c.W / 2 : c.W;
    const int out_c = c.head ? 64 : (c.out_c ? c.out_c : rows);
    const int tiles = c.n * ((c.H + kTileH - 1) / kTileH) * ((c.W + kTileW - 1) / kTileW) * c.groups * n_tiles;
    const int valid[2] = {c.head ? 38 : c.cout_g, c.head ? 19 : c.cout_g};
    const int nstore[2] = {c.head ? 40 : c.cout_g, c.head ? 24 : c.cout_g};
    const int choff[2] = {c.head ? 0 : c.out_off, c.head ? 40 : c.out_off + c.cout_g};
    if (c.pool && ((c.H | c.W) & 1)) { printf("case %s: pooling needs even H, W\n", c.name); return 1; }
    if (c.prelu && c.pool) { printf("case %s: no PReLU layer pools\n", c.name); return 1; }
    if (c.ragged && c.ext_shift < c.pool) { printf("case %s: a pooled launch has ext_shift >= 1\n", c.name); return 1; }
    rng_state = 1000003u * (ci + 1) + (exact ? 17 : 29);
    auto rnd3 = [] { rng_state = rng_state * 1664525u + 1013904223u; return (int)((rng_state >> 12) % 3) - 1; };

    // ragged extents: at the launch's output (eho, ewo) and input (ehi, ewi) resolution; the low bits of `ext` below the
    // shift are set where that keeps the input extent even under pooling, so the shift must truncate them
    std::vector<int> ext, eho(c.n, Ho), ewo(c.n, Wo), ehi(c.n, c.H), ewi(c.n, c.W);
    if (c.ragged) {
        const int lowbits = (1 << (c.ext_shift - c.pool)) - 1;
        for (int i = 0; i < c.n; ++i) {
            const int e[5][2] = {{Ho, Wo}, {Ho - 3, Wo / 2}, {Ho / 3, Wo - 1}, {1, Wo}, {Ho, 1}};
            eho[i] = std::max(1, e[i % 5][0]);
            ewo[i] = std::max(1, e[i % 5][1]);
            ext.push_back((eho[i] << c.ext_shift) | lowbits);
            ext.push_back((ewo[i] << c.ext_shift) | lowbits);
            ehi[i] = c.pool ? 2 * eho[i] : eho[i];
            ewi[i] = c.pool ? 2 * ewo[i] : ewo[i];
        }
    }
    // per-image activation scale (exact mode): fp8's amax tables give each image its own ea; fp16's overflow image
    // (each table alone also keeps every |a| 2^ea <= 256: e4m3 holds it exactly)
    const float fp8_amax0[5] = {1.0f, 0.2f, 5.0f, 2.0f, 0.75f}, fp8_amax1[5] = {0.5f, 0.15f, 7.5f, 0.f, 1.5f};
    const double fp8_s[5] = {1.0, 0.125, 4.0, 2.0, 0.5};
    std::vector<double> s_img(c.n, 1.0);
    for (int i = 0; i < c.n; ++i) {
        if (fp8) s_img[i] = fp8_s[i % 5];
        if (exact && c.ovf && i == 1) s_img[i] = 4096.0;
    }

    // operands (double values of what the device reads)
    std::vector<double> in((size_t)c.n * c.H * c.W * in_c, 0.0), in_lo(split ? in.size() : 0, 0.0);
    std::vector<double> w((size_t)taps * rows * c.cin_g, 0.0), w_lo(split ? w.size() : 0, 0.0);
    std::vector<float> bias(rows, 0.f), slope(rows, 0.f);
    std::vector<int> wexp(rows, 0);
    auto act_round = [&](double x) { return f16 ? f16_rne(x) : bf16_rne(x); };
    for (int n = 0; n < c.n; ++n)
        for (int y = 0; y < c.H; ++y)
            for (int x = 0; x < c.W; ++x)
                for (int k = 0; k < in_c; ++k) {
                    const size_t i = (((size_t)n * c.H + y) * c.W + x) * in_c + k;
                    double hi, lo = 0;
                    if (exact) {
                        hi = rnd3() * s_img[n];
                        if (split && hi != 0) lo = rnd3() * std::ldexp(s_img[n], -9);
                    } else {
                        const float v = frand();
                        hi = act_round(v);
                        if (split) lo = bf16_rne(v - hi);
                    }
                    if (y >= ehi[n] || x >= ewi[n]) hi = lo = 0;     // +0 outside the frame, as the runtime keeps it
                    in[i] = hi;
                    if (split) in_lo[i] = lo;
                }
    const float ws = 1.0f / std::sqrt((float)(taps * c.cin_g));
    const float bias_exact[7] = {0.f, 1.f, -2.f, 3.f, 0.5f, -0.25f, 2.f}, slope_exact[4] = {0.25f, -0.5f, 0.f, 1.f};
    const int wexp_fp8[6] = {0, 3, -2, 8, 5, -7};
    for (int r = 0; r < rows; ++r) {
        const int g = r / c.cout_g, co = r % c.cout_g;
        wexp[r] = wexp_fp8[r % 6];
        slope[r] = exact ? slope_exact[r % 4] : frand() * 1.2f;
        if (co >= valid[g]) continue;     // head pad rows: zero weights and bias, as the weight packer writes them
        bias[r] = exact ? (c.ovf ? (float)rnd3() * 3.f : bias_exact[(r * 5 + 2) % 7]) : frand() * 0.2f;
        for (int t = 0; t < taps; ++t)
            for (int k = 0; k < c.cin_g; ++k) {
                const size_t i = ((size_t)t * rows + r) * c.cin_g + k;
                if (exact) {
                    w[i] = rnd3();
                    if (split && w[i] != 0) w_lo[i] = rnd3() * std::ldexp(1.0, -9);
                } else {
                    const float v = frand() * 2.f * ws * 1.7f;
                    w[i] = act_round(v);
                    if (split) w_lo[i] = bf16_rne(v - w[i]);
                }
            }
    }

    // reference: r = sum(a w) + b and S = sum|a w| + |b| per pre-pool output, in double (exact in exact mode)
    std::vector<double> ref((size_t)c.n * c.H * c.W * rows), sabs(ref.size());
    double maxterm = 0;
    for (float b : bias) maxterm = std::max(maxterm, (double)std::fabs(b));
    for (int n = 0; n < c.n; ++n)
        for (int y = 0; y < c.H; ++y)
            for (int x = 0; x < c.W; ++x)
                for (int r = 0; r < rows; ++r) {
                    const int g = r / c.cout_g;
                    double acc = bias[r], sa = std::fabs(bias[r]), mt = 0;
                    for (int dy = 0; dy < c.ks; ++dy) {
                        const int yy = y + dy - pad;
                        if (yy < 0 || yy >= c.H) continue;
                        for (int dx = 0; dx < c.ks; ++dx) {
                            const int xx = x + dx - pad;
                            if (xx < 0 || xx >= c.W) continue;
                            const size_t ib = (((size_t)n * c.H + yy) * c.W + xx) * in_c + c.in_base + g * c.in_stride_g;
                            const size_t wb = ((size_t)(dy * c.ks + dx) * rows + r) * c.cin_g;
                            for (int k = 0; k < c.cin_g; ++k) {
                                const double p = in[ib + k] * w[wb + k];
                                acc += p;
                                sa += std::fabs(p);
                                mt = std::max(mt, std::fabs(p));
                                if (split) {     // A_hi W_lo + A_lo W_hi
                                    const double p1 = in[ib + k] * w_lo[wb + k], p2 = in_lo[ib + k] * w[wb + k];
                                    acc += p1 + p2;
                                    sa += std::fabs(p1) + std::fabs(p2);
                                }
                            }
                        }
                    }
                    const size_t ri = (((size_t)n * c.H + y) * c.W + x) * rows + r;
                    ref[ri] = acc;
                    sabs[ri] = sa;
                    maxterm = std::max(maxterm, mt);
                }
    if (exact) {     // the exactness argument above, checked on the operands of this case
        const double qa = *std::min_element(s_img.begin(), s_img.end()), q9 = std::ldexp(1.0, -9);
        const double qb = c.ovf ? 1.0 : 0.25;      // bias quantum
        double q = std::min(qa, qb);
        if (split) q = std::min(q, qa * q9);
        auto multiple = [](double v, double qq) { return std::fmod(v, qq) == 0; };
        bool ok = maxterm <= std::ldexp(q, 12);
        for (size_t i = 0; ok && i < in.size(); ++i) ok = multiple(in[i], qa) && (!split || multiple(in_lo[i], qa * q9));
        for (size_t i = 0; ok && i < w.size(); ++i) ok = multiple(w[i], 1.0) && (!split || multiple(w_lo[i], q9));
        for (float b : bias) ok = ok && multiple(b, qb);
        for (size_t i = 0; ok && i < sabs.size(); ++i) ok = sabs[i] <= std::ldexp(maxterm, 12);
        if (!ok) {
            printf("case %s %s: exact-mode operands break the 2^12 bound\n", c.name, fmt_name(F));
            return 1;
        }
    }

    // device operands
    std::vector<uint16_t> in_h(in.size()), in_lo_h(in_lo.size());
    for (size_t i = 0; i < in.size(); ++i) in_h[i] = f16 ? f16_rn_bits((float)in[i]) : bf16_bits(in[i]);
    for (size_t i = 0; i < in_lo.size(); ++i) in_lo_h[i] = bf16_bits(in_lo[i]);
    std::vector<uint8_t> w_bytes;
    if (fp8) {       // [taps][rows][cin] e4m3(w 2^ew[row]) in the K order of fp8_k_to_channel
        w_bytes.resize(w.size());
        for (int t = 0; t < taps; ++t)
            for (int r = 0; r < rows; ++r)
                for (int k = 0; k < c.cin_g; ++k)
                    w_bytes[((size_t)t * rows + r) * c.cin_g + k] = e4m3_rn_bits(
                        (float)std::ldexp(w[((size_t)t * rows + r) * c.cin_g + (k & ~31) + fp8_k_to_channel(k & 31)], wexp[r]));
    } else {         // bf16: [hi taps | lo taps]; fp16: [taps] binary16
        std::vector<uint16_t> wh(f16 ? w.size() : 2 * w.size(), 0);
        for (size_t i = 0; i < w.size(); ++i) {
            wh[i] = f16 ? f16_rn_bits((float)w[i]) : bf16_bits(w[i]);
            if (split) wh[w.size() + i] = bf16_bits(w_lo[i]);
        }
        w_bytes.resize(wh.size() * 2);
        memcpy(w_bytes.data(), wh.data(), w_bytes.size());
    }
    std::vector<unsigned> amax0(c.n), amax1(c.n);
    for (int i = 0; i < c.n; ++i) {
        amax0[i] = f32_bits(fp8_amax0[i % 5]);
        amax1[i] = f32_bits(fp8_amax1[i % 5]);
    }
    __nv_bfloat16* d_in = reinterpret_cast<__nv_bfloat16*>(upload(in_h));
    __nv_bfloat16* d_in_lo = split ? reinterpret_cast<__nv_bfloat16*>(upload(in_lo_h)) : nullptr;
    uint8_t* d_w = upload(w_bytes);
    float* d_bias = upload(bias);
    float* d_slope = upload(slope);
    int* d_wexp = upload(wexp);
    unsigned* d_amax0 = upload(amax0);
    unsigned* d_amax1 = upload(amax1);
    int* d_ext = c.ragged ? upload(ext) : nullptr;
    const size_t out_elems = (size_t)c.n * Ho * Wo * out_c;
    GBuf g_out = galloc(out_elems * 2), g_out_lo, g_f32[2], g_amax, g_ea, g_ovf;
    if (split) g_out_lo = galloc(out_elems * 2);
    if (c.head)
        for (int g = 0; g < 2; ++g) g_f32[g] = galloc((size_t)c.n * valid[g] * Ho * Wo * 4);
    if (fp8) { g_amax = galloc(4 * c.n); g_ea = galloc(4 * c.n); }
    if (f16) g_ovf = galloc(4 * c.n);
    GBuf* bufs[7] = {&g_out, &g_out_lo, &g_f32[0], &g_f32[1], &g_amax, &g_ea, &g_ovf};
    const int fills[7] = {0xFF, 0xFF, 0xFF, 0xFF, 0, 0x7F, 0};     // NaN words; amax and overflow 0; ea 0x7f7f7f7f

    ConvTcArgs a;
    memset(&a, 0, sizeof(a));
    a.n_img = c.n; a.H = c.H; a.W = c.W; a.ksize = c.ks; a.cin_blocks = cb;
    a.in_ch_base = c.in_base; a.in_ch_group_stride = c.in_stride_g; a.groups = c.groups;
    a.n_tile = c.N; a.n_tiles = n_tiles; a.bias = d_bias; a.relu = c.relu; a.pool = c.pool;
    a.out = reinterpret_cast<__nv_bfloat16*>(g_out.p()); a.out_cstride = out_c;
    a.out_lo = reinterpret_cast<__nv_bfloat16*>(g_out_lo.p());
    for (int g = 0; g < 2; ++g) {
        a.out_ch_off[g] = choff[g];
        a.store_ch[g] = c.head ? nstore[g] : c.N;
        a.out_f32[g] = reinterpret_cast<float*>(g_f32[g].p());
        a.f32_ch[g] = c.head ? valid[g] : 0;
    }
    a.fmt = F;
    a.slope = c.prelu ? d_slope : nullptr;
    a.ext = d_ext;
    a.ext_shift = c.ext_shift;
    if (fp8) {
        a.amax_in[0] = d_amax0;
        a.amax_in[1] = (ci & 1) ? d_amax1 : nullptr;     // every other fp8 case takes the max of two writers' tables
        a.amax_out = reinterpret_cast<unsigned*>(g_amax.p());
        a.w_exp = d_wexp;
        a.ea_out = reinterpret_cast<int*>(g_ea.p());
    }
    a.ovf_out = reinterpret_cast<unsigned*>(g_ovf.p());
    CK(conv_tc_make_maps(a, d_in, in_c, d_w, d_in_lo));

    // grid sizes, the clamped S first: it is the run checked against the reference
    std::vector<int> grids;
    for (int G : {sms, 1, 2, 3, 7, sms - 1, 2 * sms}) {
        const int eff = std::min(G, tiles);
        if (std::find(grids.begin(), grids.end(), eff) == grids.end()) grids.push_back(eff);
    }
    std::vector<std::vector<uint8_t>> base(7);
    long bad = 0;
    int printed = 0;
    double worst16 = 0, worst32 = 0;
    char gridlog[256] = "";
    for (size_t gi = 0; gi < grids.size(); ++gi) {
        for (int b = 0; b < 7; ++b) gfill(*bufs[b], fills[b]);
        CK(conv_tc_launch(a, grids[gi], 0));
        const cudaError_t e = cudaDeviceSynchronize();
        if (e != cudaSuccess) {
            printf("case %-40s %-6s N=%d: KERNEL FAILED at grid %d: %s\n", c.name, fmt_name(F), c.N, grids[gi], cudaGetErrorString(e));
            return 100;
        }
        std::vector<std::vector<uint8_t>> h(7);
        for (int b = 0; b < 7; ++b) h[b] = gread(*bufs[b]);
        if (gi > 0) {    // bit for bit the run at S, sentinels included
            long diff = 0;
            for (int b = 0; b < 7; ++b)
                for (size_t i = 0; i < h[b].size(); ++i) diff += h[b][i] != base[b][i];
            const size_t len = strlen(gridlog);
            if (len < sizeof(gridlog) - 32)
                snprintf(gridlog + len, sizeof(gridlog) - len, diff ? " %d:DIFF(%ld B)" : " %d:=", grids[gi], diff);
            bad += diff;
            continue;
        }
        base = h;
        snprintf(gridlog, sizeof(gridlog), " %d:ref", grids[0]);
        for (int b = 0; b < 7; ++b) {
            const long d = guard_damage(h[b], *bufs[b]);
            if (d && printed++ < 8) printf("  sentinel of buffer %d: %ld bytes changed\n", b, d);
            bad += d;
        }
        auto word = [&](int b, size_t i) { uint16_t v; memcpy(&v, h[b].data() + kGuard + 2 * i, 2); return v; };
        auto f32at = [&](int g, size_t i) { float v; memcpy(&v, h[2 + g].data() + kGuard + 4 * i, 4); return v; };
        auto u32at = [&](int b, int i) { uint32_t v; memcpy(&v, h[b].data() + kGuard + 4 * i, 4); return v; };
        auto fail = [&](const char* what, int n, int y, int x, int ch, double got, double lo, double hi) {
            if (printed++ < 8) printf("  bad %s: n=%d y=%d x=%d ch=%d got %.9g want [%.9g, %.9g]\n", what, n, y, x, ch, got, lo, hi);
            ++bad;
        };
        // expected value of output channel (g, co) at output pixel (n, yo, xo): f over the pool window, for r, r - e, r + e
        const double U = std::ldexp(1.0, -22);
        double coef;
        if (tc_chunked(F)) coef = c.ks == 7 ? 28 + 16 + 3 * cb * 7 : taps * 4 + 16 + 3 * cb;
        else coef = std::ceil(taps * c.cin_g / 16.0) + 16;
        auto act = [&](double v, int r) { return c.prelu ? (v > 0 ? v : (double)slope[r] * v) : (c.relu && v < 0 ? 0.0 : v); };
        struct Want { double v, lo, hi, e; };
        auto want = [&](int n, int yo, int xo, int r) {
            Want o = {-INFINITY, -INFINITY, -INFINITY, 0};
            for (int j = 0; j < (c.pool ? 4 : 1); ++j) {
                const int y = c.pool ? 2 * yo + (j >> 1) : yo, x = c.pool ? 2 * xo + (j & 1) : xo;
                const size_t ri = (((size_t)n * c.H + y) * c.W + x) * rows + r;
                const double e = exact ? 0 : U * coef * sabs[ri];
                double lo = act(ref[ri] - e, r), hi = act(ref[ri] + e, r);
                if (lo > hi) std::swap(lo, hi);
                if (ref[ri] - e < 0 && ref[ri] + e > 0) { lo = std::min(lo, 0.0); hi = std::max(hi, 0.0); }   // PReLU's kink
                o.v = std::max(o.v, act(ref[ri], r));
                o.lo = std::max(o.lo, lo);
                o.hi = std::max(o.hi, hi);
                o.e = std::max(o.e, e * (c.prelu ? std::max(1.0, (double)std::fabs(slope[r])) : 1.0));
            }
            return o;
        };
        std::vector<uint32_t> want_amax(c.n, 0);
        std::vector<int> want_ovf(c.n, 0);
        std::vector<int> owner(out_c, -1);    // output channel -> row, -1: outside the launch's slice
        for (int g = 0; g < c.groups; ++g)
            for (int co = 0; co < nstore[g]; ++co) owner[choff[g] + co] = g * c.cout_g + co;
        for (int n = 0; n < c.n; ++n)
            for (int yo = 0; yo < Ho; ++yo)
                for (int xo = 0; xo < Wo; ++xo) {
                    const bool inside = yo < eho[n] && xo < ewo[n];
                    for (int oc = 0; oc < out_c; ++oc) {
                        const size_t oi = (((size_t)n * Ho + yo) * Wo + xo) * out_c + oc;
                        const uint16_t hb = word(0, oi), lb = split ? word(1, oi) : 0;
                        const int r = owner[oc];
                        if (r < 0) {
                            if (hb != 0xFFFF || (split && lb != 0xFFFF)) fail("channel outside the slice", n, yo, xo, oc, hb, 0xFFFF, 0xFFFF);
                            continue;
                        }
                        const double got = f16 ? f16_val(hb) : bf16_val(hb);
                        if (!inside || r % c.cout_g >= valid[r / c.cout_g]) {    // beyond the frame, head pad rows: +0
                            if (hb != 0 || lb != 0) fail(inside ? "pad row" : "outside the frame", n, yo, xo, oc, got, 0, 0);
                            continue;
                        }
                        const Want wv = want(n, yo, xo, r);
                        if (exact) {
                            const double rv = r32(wv.v);     // exact: f(r) is an fp32 value
                            uint16_t eh, el = 0;
                            if (f16) eh = f16_rn_bits((float)f16_rne(rv));
                            else eh = bf16_bits(bf16_rne(rv));
                            if (split) el = bf16_bits(bf16_rne(rv - bf16_rne(rv)));
                            if (hb != eh || lb != el) fail(lb != el ? "residual word" : "word", n, yo, xo, oc, got, rv, rv);
                            if (fp8) want_amax[n] = std::max(want_amax[n], (uint32_t)(eh & 0x7fff) << 16);
                            if (f16 && (eh & 0x7c00) == 0x7c00) want_ovf[n] = 1;
                        } else {
                            bool ok;
                            double dist;
                            if (split) {
                                const double lo = bf16_val(lb);
                                const double wsl = std::ldexp(c.prelu ? std::max(std::fabs(wv.lo), std::fabs(wv.hi)) : std::fabs(wv.v), -16);
                                ok = got + lo >= wv.lo - wsl && got + lo <= wv.hi + wsl && std::fabs(lo) <= bf16_ulp(got) / 2;
                                dist = std::max(0.0, std::fabs(got + lo - wv.v) - wsl);
                            } else if (f16) {
                                ok = got >= f16_rne(r32(wv.lo)) && got <= f16_rne(r32(wv.hi));
                                dist = std::max(0.0, std::fabs(got - wv.v) - f16_ulp(got) / 2);
                            } else {
                                ok = got >= bf16_rne(r32(wv.lo)) && got <= bf16_rne(r32(wv.hi));
                                dist = std::max(0.0, std::fabs(got - wv.v) - bf16_ulp(got) / 2);
                            }
                            if (!ok) fail("interval", n, yo, xo, oc, got, wv.lo, wv.hi);
                            if (wv.e > 0) worst16 = std::max(worst16, dist / wv.e);
                        }
                    }
                    // fp32 maps (heads): channel c of group g at (n, yo, xo)
                    for (int g = 0; c.head && g < c.groups; ++g)
                        for (int co = 0; co < valid[g]; ++co) {
                            const float gf = f32at(g, (((size_t)n * valid[g] + co) * Ho + yo) * Wo + xo);
                            if (!inside) {
                                if (f32_bits(gf) != 0) fail("fp32 map outside the frame", n, yo, xo, co, gf, 0, 0);
                                continue;
                            }
                            const Want wv = want(n, yo, xo, g * c.cout_g + co);
                            if (exact) {
                                if (f32_bits(gf) != f32_bits((float)wv.v)) fail("fp32 map", n, yo, xo, co, gf, wv.v, wv.v);
                            } else {
                                if (!(gf >= r32(wv.lo) && gf <= r32(wv.hi))) fail("fp32 map interval", n, yo, xo, co, gf, wv.lo, wv.hi);
                                if (wv.e > 0) worst32 = std::max(worst32, std::fabs(gf - wv.v) / wv.e);
                            }
                        }
                }
        for (int n = 0; n < c.n; ++n) {
            if (fp8) {
                const uint32_t am = u32at(4, n);
                const int ea = (int)u32at(5, n);
                const int want_ea = fp8_exp_from_amax(std::max(amax0[n], a.amax_in[1] ? amax1[n] : 0u));
                if (am != want_amax[n]) fail("amax", n, -1, -1, -1, am, want_amax[n], want_amax[n]);
                if (ea != want_ea) fail("ea", n, -1, -1, -1, ea, want_ea, want_ea);
            }
            if (f16 && (int)u32at(6, n) != want_ovf[n]) fail("overflow flag", n, -1, -1, -1, u32at(6, n), want_ovf[n], want_ovf[n]);
        }
        if (f16 && exact && c.ovf && !want_ovf[1]) {
            printf("  case %s: image 1 does not overflow\n", c.name);
            ++bad;
        }
    }
    printf("case %-40s %-6s N=%-3d %s%s %-6s tiles %3d :%s", c.name, fmt_name(F), c.N, c.ragged ? "ragged" : "uniform",
           c.prelu ? " prelu" : "", exact ? "exact" : "random", tiles, gridlog);
    if (!exact) printf("  max|v-r|/e %.3f f32 %.3f", worst16, worst32);
    printf("  %s\n", bad ? "MISMATCH" : "OK");
    if (!exact) {
        Worst& wst = g_worst[(int)F][c.N][c.ragged][c.prelu];
        wst.w16 = std::max(wst.w16, worst16);
        wst.w32 = std::max(wst.w32, worst32);
        wst.seen = true;
    }
    cudaFree(d_in); cudaFree(d_w); cudaFree(d_bias); cudaFree(d_slope); cudaFree(d_wexp); cudaFree(d_amax0); cudaFree(d_amax1);
    if (d_in_lo) cudaFree(d_in_lo);
    if (d_ext) cudaFree(d_ext);
    for (GBuf* b : bufs)
        if (b->base) cudaFree(b->base);
    return bad ? 1 : 0;
}

}  // namespace mx

// (format, N, ragged, PReLU) of every matrix case; no CUDA call, so that the table can be read on a machine without a GPU
static int list_matrix() {
    for (const mx::MCase& c : mx::kCases) printf("case %s %d %d %d\n", mx::fmt_name(c.fmt), c.N, c.ragged, c.prelu);
    return 0;
}

static int run_matrix(int sms) {
    int fails = 0, runs = 0;
    for (size_t ci = 0; ci < sizeof(mx::kCases) / sizeof(mx::kCases[0]); ++ci) {
        const mx::MCase& c = mx::kCases[ci];
        for (int exact = 1; exact >= (c.fmt == TcFormat::kFp8 ? 1 : 0); --exact) {
            const int r = mx::run(c, (int)ci, exact, sms);
            if (r >= 100) {
                printf("aborting after kernel failure\n");
                return 3;
            }
            fails += r;
            ++runs;
        }
    }
    for (int f = 0; f < 4; ++f)
        for (int n : {128, 64, 48, 32})
            for (int pr = 0; pr < 2; ++pr)
                for (int rg = 0; rg < 2; ++rg) {
                    const mx::Worst& w = mx::g_worst[f][n][rg][pr];
                    if (w.seen)
                        printf("worst %s %d %s%s : max|v-r|/e %.3f f32 %.3f\n", mx::fmt_name((TcFormat)f), n,
                               rg ? "ragged" : "uniform", pr ? " prelu" : "", w.w16, w.w32);
                }
    printf("conv_tc matrix: %zu cases, %d case-modes, %s\n", sizeof(mx::kCases) / sizeof(mx::kCases[0]), runs,
           fails == 0 ? "ALL OK" : "FAILURES");
    return fails == 0 ? 0 : 1;
}

int main(int argc, char** argv) {
    if (argc > 1 && !strcmp(argv[1], "list")) return list_matrix();
    int dev = 0;
    CK(cudaSetDevice(dev));
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, dev));
    printf("device %s sm_%d%d, %d SMs\n", prop.name, prop.major, prop.minor, prop.multiProcessorCount);
    const int sms = prop.multiProcessorCount;
    if (argc > 1 && !strcmp(argv[1], "matrix")) return run_matrix(sms);
    const bool do_perf = argc > 1 && !strcmp(argv[1], "perf");
    const Case cases[] = {
        //  name                         n  H   W  ks g cin stride cout ntile relu pool head
        {"1x1 64->64 16x16 (aligned)", 1, 16, 16, 1, 1, 64, 64, 64, 64, 0, 0, 0},
        {"3x3 64->64 40x40", 2, 40, 40, 3, 1, 64, 64, 64, 64, 1, 0, 0},
        {"3x3 128->128 pool 32x32", 1, 32, 32, 3, 1, 128, 128, 128, 128, 1, 1, 0},
        {"7x7 2grp 128->128 30x30", 1, 30, 30, 7, 2, 128, 128, 128, 128, 1, 0, 0},
        {"7x7 2grp shared192->128 22x26", 1, 22, 26, 7, 2, 192, 0, 128, 128, 1, 0, 0},
        {"1x1 head 128->38|19 46x46", 2, 46, 46, 1, 2, 128, 128, 48, 48, 0, 0, 1},
        {"1x1 512->512 46x46 4 ntiles", 1, 46, 46, 1, 1, 512, 512, 512, 128, 1, 0, 0},
        {"3x3 64->128 odd tiles 3x40x16", 3, 40, 16, 3, 1, 64, 64, 128, 128, 1, 0, 0},     // 3 images x 3 x 2 = 18 pixel tiles
        {"7x7 2grp 128->128 1x16x16", 1, 16, 16, 7, 2, 128, 128, 128, 128, 1, 0, 0},        // two pixel tiles
        {"7x7 2grp 128->128 nt64 30x30", 1, 30, 30, 7, 2, 128, 128, 128, 64, 1, 0, 0},      // two 64-wide n-tiles per group
        {"7x7 2grp 128->128 nt32 46x46", 1, 46, 46, 7, 2, 128, 128, 128, 32, 1, 0, 0},      // batch-1 plan: four 32-wide n-tiles
        {"3x3 128->128 pool nt32 24x40", 1, 24, 40, 3, 1, 128, 128, 128, 32, 1, 1, 0},
        {"7x7 head 128->38|19 K=6272", 2, 46, 46, 7, 2, 128, 128, 48, 48, 0, 0, 1},          // fp32 outputs after a long K loop
        // 4 x 6 x 12 = 288 work items on 132 SMs: the persistent loop (ring wrap across tiles, next-tile prefetch during
        // the epilogue, accumulator reset per tile), pool over a partial last tile column (92 = 11.5 x 8)
        {"3x3 128->128 pool 4x92x92 persistent", 4, 92, 92, 3, 1, 128, 128, 128, 128, 1, 1, 0},
        // bf16x3, K-chunked: one chunk per filter row (7x7) / per channel block and term (3x3)
        {"7x7 2grp 128->128 bf16x3 nt64 23x31", 1, 23, 31, 7, 2, 128, 128, 128, 64, 1, 0, 0, 1},
        {"3x3 128->128 pool bf16x3 nt32 2x24x40", 2, 24, 40, 3, 1, 128, 128, 128, 32, 1, 1, 0, 1},
        // part of a wider buffer: channels 64..191 of 192 in (stage 1), channels 64..191 of 192 out (conv4_4_CPM)
        {"3x3 in 64..191/192 -> out 64..191/192", 2, 46, 46, 3, 1, 128, 0, 128, 128, 1, 0, 0, 0, 64, 192, 64, 192},
        // PDL-chained behind the launch that writes its input
        {"3x3 64->64 PDL behind its producer", 2, 40, 48, 3, 1, 64, 64, 64, 64, 1, 0, 0, 0, 0, 0, 0, 0, 1},
    };
    int fails = 0;
    for (const Case& c : cases) {
        // bf16, and for N <= 64 (the n-tiles of the K-chunked kernel) bf16x3 as well; split cases in bf16x3 only
        const TcFormat fmts[2] = {TcFormat::kBf16, TcFormat::kBf16x3};
        for (int f = c.split; f <= (c.n_tile <= 64 ? 1 : 0); ++f) {
            int r = run_case(c, sms, fmts[f]);
            if (r >= 100) {   // sticky CUDA error: the context is gone
                printf("aborting after kernel failure\n");
                return 3;
            }
            fails += r;
        }
    }
    printf("conv_tc: %s\n", fails == 0 ? "ALL OK" : "FAILURES");
    if (do_perf) perf(sms);
    return fails == 0 ? 0 : 1;
}
