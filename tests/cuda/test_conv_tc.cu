// Standalone GPU check of the wgmma conv kernel against a plain CPU loop (bf16-rounded operands, double
// accumulation, the interval rule of oracle/conv_check.py).  Build: see __graft_entry__.build().  Run on an H100: build/test_conv_tc [perf]
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../pytorch_realtime_multi-person_pose_estimation_b200/csrc/conv_tc.cuh"

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
    int split;          // bf16x3: hi + lo planes, three MMA terms (run K-chunked)
    int in_base, in_c;  // first input channel of group 0 / channels per input pixel (0: cin_g or cin_g * groups)
    int out_off, out_c; // first output channel of group 0 / channels per output pixel (0: groups * cout_g)
    int pdl;            // the input is written by a preceding launch (identity 1x1 conv) and this one is PDL-chained to it
};

// Every output is checked against the interval a correctly accumulated fp32 sum could round to (oracle/conv_check.py):
// r = sum(a * w) + b and S = sum|a * w| + |b| in double, e = 2^-22 * c * S with c from the kernel's accumulation
// structure, accept R(f(r - e)) <= got <= R(f(r + e)) (f = ReLU then 2x2 max, R = bf16 round-to-nearest-even).
// head: out_ch_off {0,40}, store {40,24}, f32 {38,19}; cout_g is the padded per-group Cout (n_tile).
static int run_case(const Case& c, int num_sms, int chunk = 0) {
    const int taps = c.ks * c.ks, pad = c.ks / 2;
    const int cin_blocks = c.cin_g / 64;
    const int in_c = c.in_c ? c.in_c : ((c.in_stride_g == 0) ? c.cin_g : c.cin_g * c.groups);
    const int n_tiles = c.cout_g / c.n_tile;
    const int rows = c.groups * c.cout_g;
    const int Ho = c.pool ? c.H / 2 : c.H, Wo = c.pool ? c.W / 2 : c.W;
    const int out_c = c.head ? 64 : (c.out_c ? c.out_c : rows);
    const int nterms = c.split ? 3 : 1;

    // activations: hi = bf16(x) (lo = bf16(x - hi) in split mode); weights likewise
    std::vector<float> in((size_t)c.n * c.H * c.W * in_c), in_lo(in.size(), 0.f), w((size_t)taps * rows * c.cin_g),
        w_lo(w.size(), 0.f), bias(rows);
    for (size_t i = 0; i < in.size(); ++i) {
        const float x = frand();
        in[i] = bf16r(x);
        if (c.split) in_lo[i] = bf16r(x - in[i]);
    }
    const float ws = 1.0f / std::sqrt((float)(taps * c.cin_g));
    for (size_t i = 0; i < w.size(); ++i) {
        const float x = frand() * 2.f * ws * 1.7f;
        w[i] = bf16r(x);
        if (c.split) w_lo[i] = bf16r(x - w[i]);
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
    if (c.split) {
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
    a.chunk = chunk;
    a.split = c.split;
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
        printf("case %-34s chunk=%d : KERNEL FAILED: %s\n", c.name, chunk, cudaGetErrorString(e));
        return 100;
    }
#ifdef B2P_CONV_TIMELINE
    {
        std::vector<unsigned long long> tl(64 * kTlSlots);
        CK(conv_tc_read_timeline(tl.data()));
        const char* names[10] = {"entry", "prologue done", "patch cb0", "patch cb1", "first weights", "MMAs issued", "acc complete",
                                 "tile stored", "before final sync", "exit"};
        for (int cta = 0; cta < 4; ++cta) {
            printf("  timeline %s chunk=%d CTA %d (clk since entry):", c.name, chunk, cta);
            for (int sl = 1; sl < 10; ++sl) {
                const unsigned long long v = tl[cta * kTlSlots + sl], v0 = tl[cta * kTlSlots];
                printf(" %s=%lld", names[sl], v ? (long long)(v - v0) : -1LL);
            }
            printf("\n");
        }
    }
#endif
    std::vector<__nv_bfloat16> out_h(out_elems), out_lo_h(c.split ? out_elems : 0);
    CK(cudaMemcpy(out_h.data(), d_out, out_elems * 2, cudaMemcpyDeviceToHost));
    if (c.split) CK(cudaMemcpy(out_lo_h.data(), d_out_lo, out_elems * 2, cudaMemcpyDeviceToHost));
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
                                    if (c.split) {      // A_hi W_lo + A_lo W_hi
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
    if (chunk) coef = c.ks == 7 ? 28 + 16 + nterms * cin_blocks * 7 : taps * 4 + 16 + nterms * cin_blocks;
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
                        if (c.split) {
                            const double lo = __bfloat162float(out_lo_h[oi]), wsl = std::ldexp(std::fabs(fr), -16);
                            ok = got + lo >= flo - wsl && got + lo <= fhi + wsl && std::fabs(lo) <= bf16_ulp(got) / 2;
                            dist = std::max(0.0, std::fabs(got + lo - fr) - wsl);
                        } else {
                            ok = got >= bf16_rne(flo) && got <= bf16_rne(fhi);
                            dist = std::max(0.0, std::fabs(got - fr) - bf16_ulp(got) / 2);
                        }
                        if (c.head && co >= valid[g]) ok = got == 0 && (!c.split || __bfloat162float(out_lo_h[oi]) == 0);
                        ++checked;
                        if (ef > 0) max_ratio = std::max(max_ratio, dist / ef);
                        if (!ok) {
                            if (printed++ < 5)
                                printf("  bad: n=%d y=%d x=%d ch=%d got %.9g interval [%.9g, %.9g]\n", n, yo, xo, oc, got,
                                       c.split ? flo : bf16_rne(flo), c.split ? fhi : bf16_rne(fhi));
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
                    if (c.split) memcpy(&lbits, &out_lo_h[oi], 2);
                    if (bits != 0xFFFF || lbits != 0xFFFF) ++bad;
                }
            }
    printf("case %-34s chunk=%d : %ld outputs, max|v-r|/e bf16 %.3f f32 %.3f  bad=%ld  %s\n", c.name, chunk, checked,
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

int main(int argc, char** argv) {
    int dev = 0;
    CK(cudaSetDevice(dev));
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, dev));
    printf("device %s sm_%d%d, %d SMs\n", prop.name, prop.major, prop.minor, prop.multiProcessorCount);
    const int sms = prop.multiProcessorCount;
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
        for (int chunk = c.split; chunk <= (c.n_tile <= 64 ? 1 : 0); ++chunk) {    // K-chunked accumulation (N <= 64)
            int r = run_case(c, sms, chunk);
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
