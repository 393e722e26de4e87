// Times conv_tc_kernel alone at the layer shapes of bench.py's network (batch 32, 368x368, bf16): CUDA events over 20
// launches per layer.  Built with -DB2P_CONV_TIMELINE (tools/conv_timeline.sh) it also prints, per layer, where the first
// consumer warp of the first 64 CTAs spends its clocks: waiting on the activation patch (patch_full), waiting on the
// weights (b_full), waiting for issued MMAs to complete (wgmma.wait_group), the rest of the main loop (A operand set-up
// and MMA issue) and the epilogue, averaged over those CTAs.
// Usage on an H100:  build/conv_layers [--fmt bf16|bf16x3]
#include <cstdio>
#include <cstring>
#include <vector>

#include "../pytorch_realtime_multi-person_pose_estimation_b200/csrc/conv_tc.cuh"

using namespace b2p;

#define CK(x)                                                                                   \
    do {                                                                                        \
        cudaError_t e_ = (x);                                                                   \
        if (e_ != cudaSuccess) {                                                                \
            fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_)); \
            exit(1);                                                                            \
        }                                                                                       \
    } while (0)

struct Layer {
    const char* name;
    int H, W, ks, groups, cin_g, in_stride_g, cout_g, n_tile, pool;
};

int main(int argc, char** argv) {
    TcFormat fmt = TcFormat::kBf16;
    if (argc > 2 && !strcmp(argv[1], "--fmt") && !strcmp(argv[2], "bf16x3")) fmt = TcFormat::kBf16x3;
    const bool split = fmt == TcFormat::kBf16x3;
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    printf("device %s, %d SMs, format %s\n", prop.name, prop.multiProcessorCount, split ? "bf16x3" : "bf16");
    const int n = 32;
    // bench.py's rtpose network at 368x368: trunk, stage 1 and stages 2..6 (two branches per launch)
    const Layer layers[] = {
        {"conv1_2+pool 3x3 64->64 @368", 368, 368, 3, 1, 64, 64, 64, 64, 1},
        {"conv2_2+pool 3x3 128->128 @184", 184, 184, 3, 1, 128, 128, 128, 128, 1},
        {"conv3_2 3x3 256->256 @92", 92, 92, 3, 1, 256, 256, 256, 128, 0},
        {"conv4_2 3x3 512->512 @46", 46, 46, 3, 1, 512, 512, 512, 128, 0},
        {"Mconv1 7x7 192->128 x2 @46", 46, 46, 7, 2, 192, 0, 128, 128, 0},
        {"Mconv2 7x7 128->128 x2 @46", 46, 46, 7, 2, 128, 128, 128, 128, 0},
        {"Mconv6 1x1 128->128 x2 @46", 46, 46, 1, 2, 128, 128, 128, 128, 0},
        {"Mconv7 1x1 128->48 x2 @46", 46, 46, 1, 2, 128, 128, 48, 48, 0},
    };
    for (const Layer& p : layers) {
        if (split && p.n_tile > tc_max_n_tile(fmt)) continue;
        const int taps = p.ks * p.ks;
        const int in_c = p.in_stride_g == 0 ? p.cin_g : p.cin_g * p.groups;
        const int rows = p.groups * p.cout_g;
        const int Ho = p.pool ? p.H / 2 : p.H, Wo = p.pool ? p.W / 2 : p.W;
        const size_t in_b = (size_t)n * p.H * p.W * in_c * 2, w_b = (size_t)2 * taps * rows * p.cin_g * 2;
        const size_t out_b = (size_t)n * Ho * Wo * rows * 2;
        __nv_bfloat16 *d_in, *d_w, *d_out, *d_in_lo = nullptr, *d_out_lo = nullptr;
        float* d_bias;
        CK(cudaMalloc(&d_in, in_b));
        CK(cudaMalloc(&d_w, w_b));
        CK(cudaMalloc(&d_out, out_b));
        CK(cudaMalloc(&d_bias, rows * 4));
        CK(cudaMemset(d_in, 0x3c, in_b));
        CK(cudaMemset(d_w, 0x3c, w_b));
        CK(cudaMemset(d_bias, 0, rows * 4));
        if (split) {
            CK(cudaMalloc(&d_in_lo, in_b));
            CK(cudaMalloc(&d_out_lo, out_b));
            CK(cudaMemset(d_in_lo, 0x1c, in_b));
        }
        ConvTcArgs a;
        memset(&a, 0, sizeof(a));
        a.n_img = n; a.H = p.H; a.W = p.W; a.ksize = p.ks; a.cin_blocks = p.cin_g / 64;
        a.in_ch_group_stride = p.in_stride_g; a.groups = p.groups; a.n_tile = p.n_tile; a.n_tiles = p.cout_g / p.n_tile;
        a.bias = d_bias; a.relu = 1; a.pool = p.pool; a.out = d_out; a.out_cstride = rows; a.out_lo = d_out_lo;
        a.fmt = fmt;
        for (int g = 0; g < 2; ++g) { a.out_ch_off[g] = g * p.cout_g; a.store_ch[g] = p.n_tile; }
        CK(conv_tc_make_maps(a, d_in, in_c, d_w, d_in_lo));
        for (int i = 0; i < 3; ++i) CK(conv_tc_launch(a, prop.multiProcessorCount, 0));
        CK(cudaDeviceSynchronize());
        cudaEvent_t e0, e1;
        CK(cudaEventCreate(&e0));
        CK(cudaEventCreate(&e1));
        const int iters = 20;
        CK(cudaEventRecord(e0));
        for (int i = 0; i < iters; ++i) CK(conv_tc_launch(a, prop.multiProcessorCount, 0));
        CK(cudaEventRecord(e1));
        CK(cudaDeviceSynchronize());
        float ms;
        CK(cudaEventElapsedTime(&ms, e0, e1));
        ms /= iters;
        const double flops = 2.0 * n * p.H * p.W * (double)rows * taps * p.cin_g;
        printf("layer %-32s %8.3f ms %7.1f TFLOP/s\n", p.name, ms, flops / ms * 1e-9);
#ifdef B2P_CONV_TIMELINE
        {   // the stamps of the last launch: per-CTA sums of the first consumer warp, averaged over the first 64 CTAs
            std::vector<unsigned long long> tl(64 * kTlSlots);
            CK(conv_tc_read_timeline(tl.data()));
            double pw = 0, bw = 0, dr = 0, mn = 0, ep = 0, tot = 0, tiles = 0;
            int ctas = 0;
            for (int c = 0; c < 64; ++c) {
                const unsigned long long* s = &tl[c * kTlSlots];
                if (s[kTlTiles] == 0) continue;
                ++ctas;
                pw += s[kTlPatchWait]; bw += s[kTlWeightWait]; dr += s[kTlDrain]; mn += s[kTlMain]; ep += s[kTlEpilogue];
                tot += s[kTlMain] + s[kTlEpilogue];
                tiles += s[kTlTiles];
            }
            if (ctas > 0) {
                pw /= ctas; bw /= ctas; dr /= ctas; mn /= ctas; ep /= ctas; tot /= ctas; tiles /= ctas;
                const double rest = mn - pw - bw - dr;
                printf("  clocks/CTA %.0f (%.1f tiles): patch wait %.0f (%.1f%%)  weight wait %.0f (%.1f%%)  MMA wait %.0f (%.1f%%)"
                       "  A operand + issue %.0f (%.1f%%)  epilogue %.0f (%.1f%%)\n", tot, tiles, pw, 100 * pw / tot, bw,
                       100 * bw / tot, dr, 100 * dr / tot, rest, 100 * rest / tot, ep, 100 * ep / tot);
            }
        }
#endif
        cudaEventDestroy(e0);
        cudaEventDestroy(e1);
        cudaFree(d_in); cudaFree(d_w); cudaFree(d_out); cudaFree(d_bias);
        if (d_in_lo) cudaFree(d_in_lo);
        if (d_out_lo) cudaFree(d_out_lo);
    }
    return 0;
}
