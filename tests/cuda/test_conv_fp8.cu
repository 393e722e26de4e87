// Standalone GPU check of conv_tc_fp8_kernel (the fp8 mode, DESIGN.md §2.3).  Build: see __graft_entry__.build().
//   build/test_conv_fp8        exact-integer cases: every operand in {-1, 0, 1}, every scale 2^0, so every partial sum is
//                              an integer below 2^12 and the output must equal the integer reference bit for bit whatever
//                              the accumulator does - indexing and K order with no rounding assumption
//   build/test_conv_fp8 acc    accumulator characterisation: crafted products show how many bits an e4m3 k32 wgmma keeps
//                              and whether it truncates or rounds; prints one "ACC ..." line
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../pytorch_realtime_multi-person_pose_estimation_b200/csrc/conv_tc.cuh"
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

static uint32_t rng_state = 777;
static int irand3() {      // -1, 0, 1
    rng_state = rng_state * 1664525u + 1013904223u;
    return (int)((rng_state >> 12) % 3) - 1;
}
static uint16_t f2bf(float f) {
    uint32_t u;
    memcpy(&u, &f, 4);
    u += 0x7fffu + ((u >> 16) & 1u);
    return (uint16_t)(u >> 16);
}
static float bf2f(uint16_t b) {
    uint32_t u = (uint32_t)b << 16;
    float f;
    memcpy(&f, &u, 4);
    return f;
}
template <class T> static T* upload(const std::vector<T>& v) {
    T* d = nullptr;
    CK(cudaMalloc(&d, v.size() * sizeof(T) + 16));
    CK(cudaMemcpy(d, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
    return d;
}

// One fp8 launch on the device.  x: NHWC bf16 [n][H][W][in_c]; w: fp32 [groups*cout_pad][cin_g][taps] (cout_pad rows per
// group); bias: [groups*cout_pad].  Exponents: ea = 0 for every image (amax table 448), ew = 0 for every row.
struct Fp8Conv {
    int n, H, W, ks, groups, cin_g, in_base, in_stride_g, cout_pad, n_tile, relu, pool, in_c, out_c, out_off, head, pdl;
    const int* ext;        // ragged extents (device) or null
};

static std::vector<uint8_t> pack_w(const Fp8Conv& c, const std::vector<float>& w) {
    const int taps = c.ks * c.ks, rows = c.groups * c.cout_pad;
    std::vector<uint8_t> w8((size_t)taps * rows * c.cin_g, 0);
    for (int r = 0; r < rows; ++r)
        for (int t = 0; t < taps; ++t)
            for (int k = 0; k < c.cin_g; ++k)
                w8[((size_t)t * rows + r) * c.cin_g + k] =
                    e4m3_rn_bits(w[((size_t)r * c.cin_g + (k & ~31) + fp8_k_to_channel(k & 31)) * taps + t]);
    return w8;
}

// Launches c; returns (bf16 outputs NHWC [n][Ho][Wo][out_c], fp32 head maps NCHW per group) and the amax / ea tables.
static void launch(const Fp8Conv& c, const __nv_bfloat16* d_in, __nv_bfloat16* d_out, const std::vector<float>& w,
                   const std::vector<float>& bias, float* d_f32[2], int f32_ch[2], unsigned* d_amax_out, int* d_ea,
                   int num_sms) {
    static unsigned* d_amax_in = nullptr;
    static int* d_wexp = nullptr;
    if (!d_amax_in) {
        float v = 448.f;
        unsigned b;
        memcpy(&b, &v, 4);
        CK(cudaMalloc(&d_amax_in, 4096 * 4));
        std::vector<unsigned> t(4096, b);
        CK(cudaMemcpy(d_amax_in, t.data(), t.size() * 4, cudaMemcpyHostToDevice));
        CK(cudaMalloc(&d_wexp, 4096 * 4));
        CK(cudaMemset(d_wexp, 0, 4096 * 4));
    }
    uint8_t* d_w8 = upload(pack_w(c, w));
    float* d_b = upload(bias);
    ConvTcArgs a;
    memset(&a, 0, sizeof(a));
    a.n_img = c.n; a.H = c.H; a.W = c.W; a.ksize = c.ks; a.cin_blocks = c.cin_g / 64;
    a.in_ch_base = c.in_base; a.in_ch_group_stride = c.in_stride_g; a.groups = c.groups;
    a.n_tile = c.n_tile; a.n_tiles = c.cout_pad / c.n_tile; a.bias = d_b; a.relu = c.relu; a.pool = c.pool;
    a.out = d_out; a.out_cstride = c.out_c;
    for (int g = 0; g < 2; ++g) {
        a.out_ch_off[g] = c.out_off + g * (c.head ? 40 : c.cout_pad);
        a.store_ch[g] = c.head ? (g == 0 ? 40 : 24) : c.n_tile;
        a.out_f32[g] = d_f32 ? d_f32[g] : nullptr;
        a.f32_ch[g] = d_f32 ? f32_ch[g] : 0;
    }
    a.fmt = TcFormat::kFp8; a.pdl = c.pdl;
    a.amax_in[0] = d_amax_in; a.amax_out = d_amax_out; a.w_exp = d_wexp; a.ea_out = d_ea;
    a.ext = c.ext;
    while ((a.H << a.ext_shift) < c.H) ++a.ext_shift;
    a.ext_shift += a.pool;
    CK(conv_tc_make_maps(a, d_in, c.in_c, d_w8));
    CK(conv_tc_launch(a, num_sms, 0));
    CK(cudaDeviceSynchronize());
    CK(cudaFree(d_w8));
    CK(cudaFree(d_b));
}

static int run_integer_case(const char* name, Fp8Conv c, int num_sms, const std::vector<int>& ext_hw = {}) {
    const int taps = c.ks * c.ks, pad = c.ks / 2, rows = c.groups * c.cout_pad;
    const int Ho = c.pool ? c.H / 2 : c.H, Wo = c.pool ? c.W / 2 : c.W;
    std::vector<uint16_t> x((size_t)c.n * c.H * c.W * c.in_c);
    std::vector<int> xi(x.size());
    for (size_t i = 0; i < x.size(); ++i) { xi[i] = irand3(); x[i] = f2bf((float)xi[i]); }
    std::vector<float> w((size_t)rows * c.cin_g * taps, 0.f), bias(rows, 0.f);
    const int valid[2] = {c.head ? 38 : c.cout_pad, c.head ? 19 : c.cout_pad};
    for (int g = 0; g < c.groups; ++g)
        for (int o = 0; o < valid[g]; ++o) {
            bias[g * c.cout_pad + o] = (float)(irand3() * 2);
            for (int k = 0; k < c.cin_g * taps; ++k) w[((size_t)g * c.cout_pad + o) * c.cin_g * taps + k] = (float)irand3();
        }
    __nv_bfloat16 *d_in = nullptr, *d_src = nullptr, *d_out = nullptr;
    const size_t out_elems = (size_t)c.n * Ho * Wo * c.out_c;
    CK(cudaMalloc(&d_out, out_elems * 2));
    CK(cudaMemset(d_out, 0x55, out_elems * 2));      // channels outside the launch's slice must keep this pattern
    std::vector<int> ext_d;
    int* d_ext = nullptr;
    if (!ext_hw.empty()) { d_ext = upload(ext_hw); c.ext = d_ext; }
    unsigned* d_amax;
    int* d_ea;
    CK(cudaMalloc(&d_amax, 4 * c.n));
    CK(cudaMemset(d_amax, 0, 4 * c.n));
    CK(cudaMalloc(&d_ea, 4 * c.n));
    CK(cudaMemset(d_ea, 0x7f, 4 * c.n));
    float* d_f32[2] = {nullptr, nullptr};
    int f32_ch[2] = {38, 19};
    if (c.head)
        for (int g = 0; g < 2; ++g) CK(cudaMalloc(&d_f32[g], (size_t)c.n * f32_ch[g] * Ho * Wo * 4));
    if (c.pdl) {   // producer: an fp8 1x1 identity conv d_src -> d_in (exact), this launch PDL-chained behind it
        d_src = reinterpret_cast<__nv_bfloat16*>(upload(x));
        CK(cudaMalloc(&d_in, x.size() * 2));
        Fp8Conv p = {c.n, c.H, c.W, 1, 1, c.in_c, 0, 0, c.in_c, 64, 0, 0, c.in_c, c.in_c, 0, 0, 0, nullptr};
        std::vector<float> wid((size_t)c.in_c * c.in_c, 0.f), zero(c.in_c, 0.f);
        for (int o = 0; o < c.in_c; ++o) wid[(size_t)o * c.in_c + o] = 1.f;
        unsigned* d_a2;
        CK(cudaMalloc(&d_a2, 4 * c.n));
        CK(cudaMemset(d_a2, 0, 4 * c.n));
        launch(p, d_src, d_in, wid, zero, nullptr, f32_ch, d_a2, nullptr, num_sms);
        CK(cudaFree(d_a2));
    } else {
        d_in = reinterpret_cast<__nv_bfloat16*>(upload(x));
    }
    launch(c, d_in, d_out, w, bias, c.head ? d_f32 : nullptr, f32_ch, d_amax, d_ea, num_sms);
    std::vector<uint16_t> out(out_elems);
    CK(cudaMemcpy(out.data(), d_out, out_elems * 2, cudaMemcpyDeviceToHost));
    std::vector<unsigned> amax(c.n);
    std::vector<int> ea(c.n);
    CK(cudaMemcpy(amax.data(), d_amax, 4 * c.n, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(ea.data(), d_ea, 4 * c.n, cudaMemcpyDeviceToHost));
    std::vector<std::vector<float>> f32(2);
    for (int g = 0; c.head && g < 2; ++g) {
        f32[g].resize((size_t)c.n * f32_ch[g] * Ho * Wo);
        CK(cudaMemcpy(f32[g].data(), d_f32[g], f32[g].size() * 4, cudaMemcpyDeviceToHost));
    }
    long bad = 0;
    std::vector<float> want_amax(c.n, 0.f);
    std::vector<char> written(c.out_c, 0);
    for (int img = 0; img < c.n; ++img) {
        const int eh = ext_hw.empty() ? Ho : ext_hw[2 * img] >> c.pool, ew_ = ext_hw.empty() ? Wo : ext_hw[2 * img + 1] >> c.pool;
        for (int g = 0; g < c.groups; ++g)
            for (int o = 0; o < (c.head ? (g == 0 ? 40 : 24) : c.cout_pad); ++o) {
                const int ch = c.out_off + g * (c.head ? 40 : c.cout_pad) + o;
                written[ch] = 1;
                for (int yo = 0; yo < Ho; ++yo)
                    for (int xo = 0; xo < Wo; ++xo) {
                        long best = -(1L << 40);
                        for (int py = 0; py <= c.pool; ++py)
                            for (int px = 0; px <= c.pool; ++px) {
                                const int y = yo * (1 + c.pool) + py, xx = xo * (1 + c.pool) + px;
                                long s = (long)bias[g * c.cout_pad + o];
                                for (int t = 0; t < taps; ++t) {
                                    const int iy = y + t / c.ks - pad, ix = xx + t % c.ks - pad;
                                    if (iy < 0 || iy >= c.H || ix < 0 || ix >= c.W) continue;
                                    for (int k = 0; k < c.cin_g; ++k)
                                        s += (long)xi[(((size_t)img * c.H + iy) * c.W + ix) * c.in_c + c.in_base +
                                                     g * c.in_stride_g + k] *
                                             (long)w[(((size_t)g * c.cout_pad + o) * c.cin_g + k) * taps + t];
                                }
                                if (c.relu && s < 0) s = 0;
                                best = s > best ? s : best;
                            }
                        const bool inside = yo < eh && xo < ew_;
                        const float v = inside ? (float)best : 0.f;
                        const uint16_t got = out[(((size_t)img * Ho + yo) * Wo + xo) * c.out_c + ch];
                        if (got != f2bf(v)) {
                            if (bad++ < 5) printf("  %s: img %d ch %d (%d,%d) got %g want %g\n", name, img, ch, yo, xo, bf2f(got), v);
                        }
                        want_amax[img] = std::fmax(want_amax[img], std::fabs(bf2f(f2bf(v))));
                        if (c.head && o < f32_ch[g]) {
                            const float gf = f32[g][(((size_t)img * f32_ch[g] + o) * Ho + yo) * Wo + xo];
                            if (gf != v && bad++ < 5) printf("  %s: head map g%d img %d ch %d got %g want %g\n", name, g, img, o, gf, v);
                        }
                    }
            }
        unsigned wb;
        memcpy(&wb, &want_amax[img], 4);
        if (amax[img] != wb && bad++ < 5) printf("  %s: amax img %d got %08x want %08x\n", name, img, amax[img], wb);
        if (ea[img] != 0 && bad++ < 5) printf("  %s: ea img %d = %d\n", name, img, ea[img]);
        for (int yo = 0; yo < Ho; ++yo)
            for (int xo = 0; xo < Wo; ++xo)
                for (int ch = 0; ch < c.out_c; ++ch)
                    if (!written[ch] && out[(((size_t)img * Ho + yo) * Wo + xo) * c.out_c + ch] != 0x5555 && bad++ < 5)
                        printf("  %s: channel %d outside the slice changed\n", name, ch);
    }
    printf("case %-40s %s\n", name, bad ? "FAIL" : "ok");
    cudaFree(d_in); cudaFree(d_out); cudaFree(d_amax); cudaFree(d_ea);
    if (d_src) cudaFree(d_src);
    if (d_ext) cudaFree(d_ext);
    for (auto p : d_f32) if (p) cudaFree(p);
    return bad ? 1 : 0;
}

// Accumulator characterisation on a 1x1 conv, 64 input channels (two k32 steps), one 8 x 16 tile, 32 output channels,
// every scale 2^0.  Pixel p (= j) and output channel n give one experiment each; the results are the exact fp32 values of
// the head map.  Products of 2^-j use a = 2^-min(j, 9), w = 2^-(j - min(j, 9)) (e4m3 reaches 2^-9).
static int characterise(int num_sms) {
    const int n = 1, H = 16, W = 8, C = 64, N = 32, P = H * W;
    std::vector<uint16_t> x((size_t)P * C, 0);
    std::vector<float> w((size_t)N * C, 0.f), bias(N, 0.f);
    auto pw = [](int e) { return std::ldexp(1.0f, -e); };
    // input channel 0 = 1; channels 1, 2, 3 and 33 carry 2^-min(j, 9) at pixel j
    for (int p = 0; p < P; ++p) {
        const int j = p;
        x[(size_t)p * C + 0] = f2bf(1.f);
        const float s = pw(j < 9 ? j : 9);
        for (int ch : {1, 2, 3, 33}) x[(size_t)p * C + ch] = f2bf(s);
    }
    // pixels 10 .. 18 carry 2^-(p - 9) and are read by the "deep" rows, whose weights are 2^-9: small term 2^-p again
    for (int p = 10; p < P; ++p)
        for (int ch : {1, 2, 3, 33}) x[(size_t)p * C + ch] = f2bf(pw(p - 9 < 9 ? p - 9 : 9));
    // output rows: A (0): 1 + a1 w (w = 1) ; A' (16): 1 + a1 * 2^-9
    //              B (1): 1 + a1 + a2 (two equal small terms) ; B' (17)
    //              C (2): 1 + a33 (the small term in the second k32 step) ; C' (18)
    //              D (3): 1 - a1 ; D' (19)
    //              E (4): 1 + a1 + 2 a2 (3 * small: with small = 2^-(bits + 2), 0.75 of the last kept bit) ; E' (20)
    for (int deep = 0; deep < 2; ++deep) {
        const float m = deep ? pw(9) : 1.f;
        const int r = deep ? 16 : 0;
        for (int k = 0; k < 5; ++k) w[(size_t)(r + k) * C + 0] = 1.f;
        w[(size_t)(r + 0) * C + 1] = m;
        w[(size_t)(r + 1) * C + 1] = m; w[(size_t)(r + 1) * C + 2] = m;
        w[(size_t)(r + 2) * C + 33] = m;
        w[(size_t)(r + 3) * C + 1] = -m;
        w[(size_t)(r + 4) * C + 1] = m; w[(size_t)(r + 4) * C + 2] = m * 2.f;
    }
    __nv_bfloat16* d_in = reinterpret_cast<__nv_bfloat16*>(upload(x));
    float* d_f32[2];
    int f32_ch[2] = {N, 0};
    CK(cudaMalloc(&d_f32[0], (size_t)N * P * 4));
    d_f32[1] = nullptr;
    unsigned* d_amax;
    CK(cudaMalloc(&d_amax, 4));
    Fp8Conv c = {n, H, W, 1, 1, C, 0, 0, N, 32, 0, 0, C, 32, 0, 0, 0, nullptr};
    launch(c, d_in, nullptr, w, bias, d_f32, f32_ch, d_amax, nullptr, num_sms);
    std::vector<float> r((size_t)N * P);
    CK(cudaMemcpy(r.data(), d_f32[0], r.size() * 4, cudaMemcpyDeviceToHost));
    auto at = [&](int row, int j) { return (double)r[(size_t)row * P + j]; };
    // the small term of pixel j: 2^-j for the shallow rows (j <= 9), 2^-(9 + min(j - 9, 9)) for the deep rows
    int bits = -1, bits_cross = -1;
    bool per_term = false, rounds = false;
    printf("  e   1+t          1+2t         1+t(step 2)  1-t          1+3t      (t = 2^-e)\n");
    for (int e = 1; e <= 18; ++e) {
        const int row = e > 9 ? 16 : 0, pix = e;       // pixel e's small term is 2^-e in the row set of its depth
        const double t = std::ldexp(1.0, -e);
        const double A = at(row + 0, pix), B = at(row + 1, pix), Cc = at(row + 2, pix), D = at(row + 3, pix), E = at(row + 4, pix);
        printf("  %2d  %.9g  %.9g  %.9g  %.9g  %.9g\n", e, A, B, Cc, D, E);
        if (A == 1 + t && bits == e - 1) bits = e;
        if (bits == -1 && e == 1 && A == 1 + t) bits = 1;
        if (Cc == 1 + t && bits_cross == e - 1) bits_cross = e;
        if (bits_cross == -1 && e == 1 && Cc == 1 + t) bits_cross = 1;
    }
    if (bits > 0 && bits < 18) {
        const int e = bits + 1, pix = e, row = e > 9 ? 16 : 0;
        per_term = at(row + 1, pix) == 1.0;                       // two halves of the last kept bit were both dropped
        const int e2 = bits + 2;                                  // 1 + 3 * 2^-(bits+2) = 1 + 0.75 of the last kept bit
        if (e2 <= 18) rounds = at(e2 > 9 ? 20 : 4, e2) > 1.0;
    }
    printf("ACC bits=%d cross_step_bits=%d per_term=%d rounds=%d\n", bits, bits_cross, per_term ? 1 : 0, rounds ? 1 : 0);
    cudaFree(d_in); cudaFree(d_f32[0]); cudaFree(d_amax);
    return 0;
}

int main(int argc, char** argv) {
    CK(cudaSetDevice(0));
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    printf("device %s sm_%d%d, %d SMs\n", prop.name, prop.major, prop.minor, prop.multiProcessorCount);
    const int sms = prop.multiProcessorCount;
    if (argc > 1 && !strcmp(argv[1], "acc")) return characterise(sms);
    int fails = 0;
    //                     n  H   W  ks g  cin base stride cout ntile relu pool in_c out_c off head pdl
    fails += run_integer_case("1x1 64->64 N64", {1, 16, 16, 1, 1, 64, 0, 0, 64, 64, 0, 0, 64, 64, 0, 0, 0, nullptr}, sms);
    fails += run_integer_case("3x3 128->64 N64 relu 2x40x24", {2, 40, 24, 3, 1, 128, 0, 0, 64, 64, 1, 0, 128, 64, 0, 0, 0, nullptr}, sms);
    fails += run_integer_case("3x3 64->64 N32 pool 24x40", {1, 24, 40, 3, 1, 64, 0, 0, 64, 32, 1, 1, 64, 64, 0, 0, 0, nullptr}, sms);
    fails += run_integer_case("7x7 2grp 128->64 N64 23x31", {1, 23, 31, 7, 2, 128, 0, 128, 64, 64, 1, 0, 256, 128, 0, 0, 0, nullptr}, sms);
    fails += run_integer_case("7x7 2grp shared 192->64 N32 22x26", {1, 22, 26, 7, 2, 192, 0, 0, 64, 32, 1, 0, 192, 128, 0, 0, 0, nullptr}, sms);
    fails += run_integer_case("1x1 head 128->38|19 N48 2x46x46", {2, 46, 46, 1, 2, 128, 0, 128, 48, 48, 0, 0, 256, 64, 0, 1, 0, nullptr}, sms);
    fails += run_integer_case("7x7 head 128->38|19 N48 1x20x20", {1, 20, 20, 7, 2, 128, 0, 128, 48, 48, 0, 0, 256, 64, 0, 1, 0, nullptr}, sms);
    fails += run_integer_case("3x3 in 64..191/192 -> out 64..127/192", {2, 30, 30, 3, 1, 128, 64, 0, 64, 64, 1, 0, 192, 192, 64, 0, 0, nullptr}, sms);
    fails += run_integer_case("3x3 128->64 N64 PDL-chained", {2, 32, 24, 3, 1, 128, 0, 0, 64, 64, 1, 0, 128, 64, 0, 0, 1, nullptr}, sms);
    fails += run_integer_case("3x3 64->64 N64 pool ragged 3x48x40", {3, 48, 40, 3, 1, 64, 0, 0, 64, 64, 1, 1, 64, 64, 0, 0, 0, nullptr}, sms,
                              {48, 40, 24, 16, 32, 40});
    fails += run_integer_case("1x1 512->64 N64 4 images", {4, 46, 46, 1, 1, 512, 0, 0, 64, 64, 1, 0, 512, 64, 0, 0, 0, nullptr}, sms);
    printf(fails ? "%d CASES FAILED\n" : "ALL OK\n", fails);
    return fails ? 1 : 0;
}
