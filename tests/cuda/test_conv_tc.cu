// Standalone GPU check of the wgmma conv kernel against a plain CPU loop (bf16-rounded operands, double
// accumulation).  Build: see __graft_entry__.build().  Run on an H100: build/test_conv_tc [perf]
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

struct Case {
    const char* name;
    int n, H, W, ks, groups, cin_g, in_stride_g, cout_g, n_tile, relu, pool, head;
};

// head: out_ch_off {0,40}, store {40,24}, f32 {38,19}; cout_g is the padded per-group Cout (n_tile).
static int run_case(const Case& c, int num_sms, int chunk = 0) {
    const int taps = c.ks * c.ks, pad = c.ks / 2;
    const int cin_blocks = c.cin_g / 64;
    const int in_c = (c.in_stride_g == 0) ? c.cin_g : c.cin_g * c.groups;
    const int n_tiles = c.cout_g / c.n_tile;
    const int rows = c.groups * c.cout_g;
    const int Ho = c.pool ? c.H / 2 : c.H, Wo = c.pool ? c.W / 2 : c.W;
    const int out_c = c.head ? 64 : rows;

    std::vector<float> in((size_t)c.n * c.H * c.W * in_c), w((size_t)taps * rows * c.cin_g), bias(rows);
    for (auto& v : in) v = bf16r(frand());
    const float ws = 1.0f / std::sqrt((float)(taps * c.cin_g));
    for (auto& v : w) v = bf16r(frand() * 2.f * ws * 1.7f);
    for (auto& v : bias) v = frand() * 0.2f;
    const int valid[2] = {c.head ? 38 : c.cout_g, c.head ? 19 : c.cout_g};
    if (c.head)  // padded rows carry zero weights/bias, as the weight packer does
        for (int g = 0; g < c.groups; ++g)
            for (int r = valid[g]; r < c.cout_g; ++r) {
                bias[g * c.cout_g + r] = 0.f;
                for (int t = 0; t < taps; ++t)
                    for (int k = 0; k < c.cin_g; ++k) w[((size_t)t * rows + g * c.cout_g + r) * c.cin_g + k] = 0.f;
            }

    // the weight tensor map spans 2*taps slices (value + residual planes); only the first `taps` are used here
    std::vector<__nv_bfloat16> in_h(in.size()), w_h(2 * w.size(), __float2bfloat16(0.f));
    for (size_t i = 0; i < in.size(); ++i) in_h[i] = __float2bfloat16(in[i]);
    for (size_t i = 0; i < w.size(); ++i) w_h[i] = __float2bfloat16(w[i]);

    __nv_bfloat16 *d_in, *d_w, *d_out;
    float *d_bias, *d_f32[2] = {nullptr, nullptr};
    CK(cudaMalloc(&d_in, in_h.size() * 2));
    CK(cudaMalloc(&d_w, w_h.size() * 2));
    CK(cudaMalloc(&d_bias, bias.size() * 4));
    const size_t out_elems = (size_t)c.n * Ho * Wo * out_c;
    CK(cudaMalloc(&d_out, out_elems * 2));
    CK(cudaMemset(d_out, 0xFF, out_elems * 2));
    CK(cudaMemcpy(d_in, in_h.data(), in_h.size() * 2, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_w, w_h.data(), w_h.size() * 2, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_bias, bias.data(), bias.size() * 4, cudaMemcpyHostToDevice));
    if (c.head)
        for (int g = 0; g < 2; ++g) CK(cudaMalloc(&d_f32[g], (size_t)c.n * valid[g] * c.H * c.W * 4));

    ConvTcArgs a;
    memset(&a, 0, sizeof(a));
    a.n_img = c.n; a.H = c.H; a.W = c.W; a.ksize = c.ks; a.cin_blocks = cin_blocks;
    a.in_ch_base = 0; a.in_ch_group_stride = c.in_stride_g; a.groups = c.groups;
    a.n_tile = c.n_tile; a.n_tiles = n_tiles; a.bias = d_bias; a.relu = c.relu; a.pool = c.pool;
    a.out = d_out; a.out_cstride = out_c;
    for (int g = 0; g < 2; ++g) {
        a.out_ch_off[g] = c.head ? (g == 0 ? 0 : 40) : g * c.cout_g;
        a.store_ch[g] = c.head ? (g == 0 ? 40 : 24) : c.n_tile;
        a.out_f32[g] = d_f32[g];
        a.f32_ch[g] = c.head ? valid[g] : 0;
    }
    a.chunk = chunk;
    CK(conv_tc_make_maps(a, d_in, in_c, d_w));
    CK(conv_tc_launch(a, num_sms, 0));
    cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) {
        printf("case %-28s chunk=%d : KERNEL FAILED: %s\n", c.name, chunk, cudaGetErrorString(e));
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
    std::vector<__nv_bfloat16> out_h(out_elems);
    CK(cudaMemcpy(out_h.data(), d_out, out_elems * 2, cudaMemcpyDeviceToHost));
    std::vector<float> f32_h[2];
    if (c.head)
        for (int g = 0; g < 2; ++g) {
            f32_h[g].resize((size_t)c.n * valid[g] * c.H * c.W);
            CK(cudaMemcpy(f32_h[g].data(), d_f32[g], f32_h[g].size() * 4, cudaMemcpyDeviceToHost));
        }

    // CPU reference
    std::vector<float> ref((size_t)c.n * c.H * c.W * rows);
    for (int n = 0; n < c.n; ++n)
        for (int y = 0; y < c.H; ++y)
            for (int x = 0; x < c.W; ++x)
                for (int g = 0; g < c.groups; ++g)
                    for (int co = 0; co < c.cout_g; ++co) {
                        double acc = bias[g * c.cout_g + co];
                        for (int dy = 0; dy < c.ks; ++dy) {
                            int yy = y + dy - pad;
                            if (yy < 0 || yy >= c.H) continue;
                            for (int dx = 0; dx < c.ks; ++dx) {
                                int xx = x + dx - pad;
                                if (xx < 0 || xx >= c.W) continue;
                                const float* ip = &in[((size_t)(n * c.H + yy) * c.W + xx) * in_c + g * c.in_stride_g];
                                const float* wp = &w[((size_t)(dy * c.ks + dx) * rows + g * c.cout_g + co) * c.cin_g];
                                float s = 0.f;
                                for (int k = 0; k < c.cin_g; ++k) s += ip[k] * wp[k];
                                acc += s;
                            }
                        }
                        float v = (float)acc;
                        if (c.relu) v = v > 0.f ? v : 0.f;
                        ref[((size_t)(n * c.H + y) * c.W + x) * rows + g * c.cout_g + co] = v;
                    }
    double max_err = 0, max_ref = 0, max_err32 = 0;
    long bad = 0;
    for (int n = 0; n < c.n; ++n)
        for (int yo = 0; yo < Ho; ++yo)
            for (int xo = 0; xo < Wo; ++xo)
                for (int g = 0; g < c.groups; ++g) {
                    const int nstore = c.head ? (g == 0 ? 40 : 24) : c.cout_g;
                    for (int co = 0; co < nstore; ++co) {
                        float r;
                        if (c.pool) {
                            r = -1e30f;
                            for (int j = 0; j < 4; ++j) {
                                float t = ref[((size_t)(n * c.H + 2 * yo + (j >> 1)) * c.W + 2 * xo + (j & 1)) * rows +
                                              g * c.cout_g + co];
                                r = t > r ? t : r;
                            }
                        } else
                            r = ref[((size_t)(n * c.H + yo) * c.W + xo) * rows + g * c.cout_g + co];
                        const int oc = (c.head ? (g == 0 ? 0 : 40) : g * c.cout_g) + co;
                        float got = __bfloat162float(out_h[((size_t)(n * Ho + yo) * Wo + xo) * out_c + oc]);
                        double err = std::fabs((double)got - r);
                        if (!(err <= 0.02 + 0.01 * std::fabs(r))) ++bad;
                        if (err > max_err || std::isnan(got)) max_err = std::isnan(got) ? 1e9 : err;
                        if (std::fabs(r) > max_ref) max_ref = std::fabs(r);
                        if (c.head && co < valid[g]) {
                            float g32 = f32_h[g][((size_t)(n * valid[g] + co) * c.H + yo) * c.W + xo];
                            double e32 = std::fabs((double)g32 - r);
                            if (e32 > max_err32 || std::isnan(g32)) max_err32 = std::isnan(g32) ? 1e9 : e32;
                            if (!(e32 <= 2e-3 + 2e-3 * std::fabs(r))) ++bad;
                        }
                    }
                }
    printf("case %-28s chunk=%d : max|err| bf16 %.5f  f32 %.3e  (max|ref| %.3f)  bad=%ld  %s\n", c.name, chunk, max_err,
           max_err32, max_ref, bad, bad == 0 ? "OK" : "MISMATCH");
    cudaFree(d_in); cudaFree(d_w); cudaFree(d_bias); cudaFree(d_out);
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
    };
    int fails = 0;
    for (const Case& c : cases) {
        for (int chunk = 0; chunk <= (c.n_tile <= 64 ? 1 : 0); ++chunk) {    // K-chunked accumulation (N <= 64)
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
