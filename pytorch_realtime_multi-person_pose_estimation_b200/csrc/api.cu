// C-ABI of libb200pose.so (include/b200pose.h): network object, post-processing object, fused inference and the
// legacy pafprocess surface.  Host-side runtime only; the kernels live in conv_tc.cu, conv_misc.cu, postprocess.cu.
#include <array>
#include <atomic>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <list>
#include <map>
#include <memory>
#include <set>
#include <mutex>
#include <string>
#include <tuple>
#include <utility>
#include <vector>

#include "../../include/b200pose.h"
#include "aug.cuh"
#include "coco_eval.cuh"
#include "conv_misc.cuh"
#include "conv_tc.cuh"
#include "f16_core.h"
#include "draw.cuh"
#include "frames.cuh"
#include "gt.cuh"
#include "jpeg.cuh"
#include "jpeg_enc.cuh"
#include "png_enc.cuh"
#include "png.cuh"
#include "fp8_core.h"
#include "postprocess.cuh"
#include "refine_core.h"
#include "resize.cuh"
#include "tta.cuh"

using namespace b2p;

namespace {

thread_local std::string g_err;
std::atomic<long> g_launches{0};

int fail(const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_err = buf;
    return 1;
}
// fail() for a CUDA call that failed: also clears the thread's last CUDA error, which the launch wrappers report
// (cudaGetLastError), so that the error does not fail a later call.  Sticky errors cannot be cleared.
template <class... A> int cuda_fail(const char* fmt, A... args) {
    cudaGetLastError();
    return fail(fmt, args...);
}
#define CU(x)                                                                                       \
    do {                                                                                            \
        cudaError_t e_ = (x);                                                                       \
        if (e_ != cudaSuccess) return cuda_fail("%s failed: %s (%s:%d)", #x, cudaGetErrorString(e_), __FILE__, __LINE__); \
    } while (0)

// Counts the launches of a kernel wrapper that returned e.
int launched(cudaError_t e, const char* what, int launches = 1) {
    if (e != cudaSuccess) return cuda_fail("%s: %s", what, cudaGetErrorString(e));
    g_launches += launches;
    return 0;
}

// ---------------------------------------------------------------- layer table (rtpose_vgg.py:69-127)
struct ConvSpec { int cin, cout, ks; };
const ConvSpec kTrunk[12] = {{3, 64, 3},    {64, 64, 3},   {64, 128, 3},  {128, 128, 3}, {128, 256, 3}, {256, 256, 3},
                             {256, 256, 3}, {256, 256, 3}, {256, 512, 3}, {512, 512, 3}, {512, 256, 3}, {256, 128, 3}};
const bool kPoolAfter[12] = {false, true, false, true, false, false, false, true, false, false, false, false};
constexpr int kPaf = 38, kHeat = 19, kFeat = 128, kCat = kPaf + kHeat + kFeat;

constexpr int kStages = 6;     // refinement stages of the network; a forward may stop after any of them
// physical channel of the bf16 concat buffer [paf 0..37, pad, heat 40..58, pad, feat 64..191] for reference
// concat channel c of torch.cat([paf, heat, feat], 1) (rtpose_vgg.py:165)
int cat_phys(int c) { return c < kPaf ? c : (c < kPaf + kHeat ? c + 2 : c + 7); }

// ---------------------------------------------------------------- OpenPose_Model (lib/network/openpose.py), DESIGN §2.11
// Trunk: rtpose's twelve convs, with a per-channel PReLU instead of the ReLU after conv4_2, conv4_3_CPM and conv4_4_CPM.
// Then l2 PAF stages and l1 heat-map stages, one after the other (stage t of the net = L2 stage t + 1 for t < l2, else
// L1 stage t - l2 + 1).  A stage is five dense blocks of three 3x3 convs Mconv{b}_{0,1,2} whose outputs are concatenated,
// a 1x1 Mconv6 and the 1x1 head Mconv7; every conv but Mconv7 is followed by a PReLU.  Stage inputs: the features (L2
// stage 1), cat[features, paf] (L2 stages >= 2, L1 stage 1), cat[features, heat, paf] (L1 stages >= 2).
enum Nonlin { kNoAct, kRelu, kPrelu };
constexpr int kOpMaxStages = 12;
bool op_valid(int l2, int l1) { return l2 >= 1 && l1 >= 1 && l2 + l1 <= kOpMaxStages; }
struct OpStage {
    bool paf, first;                  // PAF (L2) stage; first stage of its branch (96 inner channels)
    int in, inner, innerout, out;     // StageBlock's channels
};
OpStage op_stage(int l2, int t) {
    const bool paf = t < l2, first = t == 0 || t == l2;
    const int in = t == 0 ? kFeat : (paf || first ? kFeat + kPaf : kFeat + kHeat + kPaf);
    return {paf, first, in, first ? 96 : 128, first ? 256 : 512, paf ? kPaf : kHeat};
}

// Input channel permutation of a tensor-core layer: reference channel c of its input -> channel of the buffer it reads.
enum InPerm {
    kPermNone,
    kPermRtposeCat,      // torch.cat([paf, heat, feat]) in the concat buffer (cat_phys)
    kPermFeatPaf,        // OpenPose_Model: torch.cat([features, paf]) in the concat buffer
    kPermFeatHeatPaf,    // ... torch.cat([features, heat, paf])
    kPermSlots,          // a dense block's cat of three outputs of `slot` channels, one 128-channel slot each
};
int perm_phys(InPerm perm, int slot, int c) {
    switch (perm) {
        case kPermNone: break;
        case kPermRtposeCat: return cat_phys(c);
        case kPermFeatPaf: return c < kFeat ? 64 + c : c - kFeat;
        case kPermFeatHeatPaf: return c < kFeat ? 64 + c : (c < kFeat + kHeat ? 40 + c - kFeat : c - kFeat - kHeat);
        case kPermSlots: return (c / slot) * 128 + c % slot;
    }
    return c;
}

uint16_t f2bf(float f) {
    uint32_t u;
    memcpy(&u, &f, 4);
    if ((u & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((u >> 16) | 0x40);
    u += 0x7fffu + ((u >> 16) & 1u);
    return (uint16_t)(u >> 16);
}

float bf2f(uint16_t b) {
    uint32_t u = (uint32_t)b << 16;
    float f;
    memcpy(&f, &u, 4);
    return f;
}

// Owners of the CUDA resources of the net and post objects: each releases what it holds when it is destroyed, so that a
// call that fails part-way leaks nothing.  Move-only.
template <class T> struct DevBuf {      // device memory
    T* p = nullptr;
    size_t n = 0;
    DevBuf() = default;
    DevBuf(DevBuf&& o) noexcept : p(std::exchange(o.p, nullptr)), n(std::exchange(o.n, 0)) {}
    ~DevBuf() { release(); }
    cudaError_t ensure(size_t count) {  // room for count elements: a larger request frees the old buffer first
        if (count <= n) return cudaSuccess;
        release();
        cudaError_t e = cudaMalloc(&p, count * sizeof(T));
        if (e == cudaSuccess) n = count;
        return e;
    }
    void release() { if (p) cudaFree(p); p = nullptr; n = 0; }
};

template <class T> struct HostBuf {     // pinned host memory
    T* p = nullptr;
    HostBuf() = default;
    HostBuf(HostBuf&& o) noexcept : p(std::exchange(o.p, nullptr)) {}
    ~HostBuf() { if (p) cudaFreeHost(p); }
    cudaError_t alloc(size_t count, unsigned flags) { return cudaHostAlloc(&p, count * sizeof(T), flags); }   // once
};

template <class H, cudaError_t (*Destroy)(H)> struct Handle {     // created through &h; reads as the raw handle
    H h = nullptr;
    Handle() = default;
    Handle(Handle&& o) noexcept : h(std::exchange(o.h, nullptr)) {}
    ~Handle() { if (h) Destroy(h); }
    operator H() const { return h; }
};
using Event = Handle<cudaEvent_t, cudaEventDestroy>;
using Stream = Handle<cudaStream_t, cudaStreamDestroy>;
using GraphExec = Handle<cudaGraphExec_t, cudaGraphExecDestroy>;

struct TcLayer {            // one grouped tensor-core launch
    int ks, cin_blocks, groups, n_tile, n_tiles, relu, pool;
    bool prelu = false;           // PReLU epilogue (OpenPose_Model) with `slope`, instead of `relu`
    double macs_per_pixel = 0;    // algorithmic (unpadded) MACs per output pixel, all groups
    DevBuf<float> bias;           // [groups*n_tiles*n_tile]
    DevBuf<float> slope;          // PReLU slopes, laid out like the bias (pad rows 0)
    std::vector<int> convs;       // state-dict conv per group
    InPerm perm = kPermNone;      // input channels permuted (perm_phys) ...
    int slot = 0;                 // ... kPermSlots: channels per slot
    // packed weights per encoding (TcWeights, tc_format.h), rows groups*n_tiles*n_tile of cin_blocks*64 channels; see
    // ensure_packed for when each is packed
    DevBuf<unsigned char> w[kNumTcWeights];
    DevBuf<int> w_exp;            // e4m3: ew per row (device)
    std::vector<int> h_w_exp;     // ... and its host copy (b200pose_net_debug_fp8)
};

// Activation buffers (the buffer ids of the test hooks): channels per pixel and spatial divisor.
enum Act { T1, T2, T3, T4, T5A, T5B, T6, T7, T8, T9, CAT, BRA, BRB, BR512, kNumAct };
constexpr int kMaxRagged = 1024;      // images of one ragged forward (flip: 2 per frame)
const int kActC[kNumAct] = {64, 64, 128, 128, 256, 256, 256, 512, 512, 256, 192, 256, 256, 1024};
const int kActDiv[kNumAct] = {1, 2, 2, 4, 4, 4, 8, 8, 8, 8, 8, 8, 8, 8};

// One launch of a tensor-core plan: the buffers it reads and writes and its channel slices of them.  A launch
// runs at the resolution of its input buffer.
struct Wiring {
    int in, in_base, in_group_stride;   // input buffer, first channel of group 0, channel offset of group 1
    int out, out_off[2], store[2];      // output buffer; per group: first channel, channels stored per n-tile
    bool maps;                          // stage head: also writes the stage's fp32 PAF (group 0) and heatmap (group 1)
};
// trunk (conv1_1 runs on CUDA cores before the plan)
const Wiring kTrunkWiring[11] = {
    // in  base stride out   out_off   store
    {T1,   0, 0,      T2,   {0, 0},   {64, 0}},      // conv1_2 + pool
    {T2,   0, 0,      T3,   {0, 0},   {128, 0}},     // conv2_1
    {T3,   0, 0,      T4,   {0, 0},   {128, 0}},     // conv2_2 + pool
    {T4,   0, 0,      T5A,  {0, 0},   {128, 0}},     // conv3_1
    {T5A,  0, 0,      T5B,  {0, 0},   {128, 0}},     // conv3_2
    {T5B,  0, 0,      T5A,  {0, 0},   {128, 0}},     // conv3_3
    {T5A,  0, 0,      T6,   {0, 0},   {128, 0}},     // conv3_4 + pool
    {T6,   0, 0,      T7,   {0, 0},   {128, 0}},     // conv4_1
    {T7,   0, 0,      T8,   {0, 0},   {128, 0}},     // conv4_2
    {T8,   0, 0,      T9,   {0, 0},   {128, 0}},     // conv4_3_CPM
    {T9,   0, 0,      CAT,  {64, 0},  {128, 0}},     // conv4_4_CPM -> feature slice of the concat buffer
};
// Stages: both branches run as one two-group launch (group 0 = PAF, group 1 = heatmap); each group reads and writes
// its own half of bra / brb / br512, and the head writes the PAF and heatmap slices of the concat buffer (DESIGN §1).
const Wiring kStage1Wiring[5] = {
    {CAT,   64, 0,    BRA,   {0, 128}, {128, 128}},       // the features only
    {BRA,   0,  128,  BRB,   {0, 128}, {128, 128}},
    {BRB,   0,  128,  BRA,   {0, 128}, {128, 128}},
    {BRA,   0,  128,  BR512, {0, 512}, {128, 128}},
    {BR512, 0,  512,  CAT,   {0, 40},  {40, 24}, true},
};
const Wiring kStageWiring[7] = {     // stages 2 .. 6
    {CAT,   0,  0,    BRA,   {0, 128}, {128, 128}},       // all 192 channels
    {BRA,   0,  128,  BRB,   {0, 128}, {128, 128}},
    {BRB,   0,  128,  BRA,   {0, 128}, {128, 128}},
    {BRA,   0,  128,  BRB,   {0, 128}, {128, 128}},
    {BRB,   0,  128,  BRA,   {0, 128}, {128, 128}},
    {BRA,   0,  128,  BRB,   {0, 128}, {128, 128}},
    {BRB,   0,  128,  CAT,   {0, 40},  {40, 24}, true},
};
// ---------------------------------------------------------------- the architecture of a net
// A conv in state_dict order and the nonlinearity after it.  Its tensors are the weight, the bias and, for a PReLU
// conv, the slopes.
struct ArchConv { ConvSpec s; Nonlin act; };

// One tensor-core launch, in launch order (conv1_1 runs on CUDA cores before them).  Its ReLU or PReLU is its convs'.
struct ArchLayer {
    int stage;                // 0 = the trunk; a forward of k stages runs the layers of stages 0 .. k
    std::vector<int> convs;   // conv per group
    int n_tile, pool;
    InPerm perm;
    Wiring wiring;
    int map0;                 // stage head: the fp32 map group 0 writes (group 1: map0 + 1); -1 otherwise
};

// Everything the runtime knows about a net's architecture, built once when the net is created.
struct NetArch {
    std::string name;                   // as the refusals print it
    int l2 = 0, l1 = 0;                 // OpenPose_Model's L2 / L1 stage counts; 0 for rtpose
    int stages = 0;                     // refinement stages; a net runs all of them unless set_stages asks for fewer
    std::vector<ArchConv> convs;        // state_dict order
    std::vector<ArchLayer> layers;      // launch order
    int act_c[kNumAct];                 // channels per pixel of each activation buffer
    bool zero_pads[kNumAct] = {};       // buffers with pad lanes no launch writes: zeroed when a plan is built
    // channels of each stage map (outputs[] entries, saved_for_loss order): rtpose [paf_1, heat_1, ..., paf_6, heat_6];
    // OpenPose_Model [paf_1 .. paf_l2, heat_1 .. heat_l1]
    int map_ch[12];
    // by stage count k, for every k a forward of the net may run: the stage maps 0 .. maps-1 it writes and, among
    // them, the final PAF and heat map
    struct { int maps, paf, heat; } out[kOpMaxStages + 1] = {};
};

// The trunk of both architectures: rtpose's twelve convs, PReLU after those from prelu_from on, and the eleven
// tensor-core layers of conv1_2 .. conv4_4_CPM.
NetArch trunk_arch(int prelu_from) {
    NetArch a;
    for (int i = 0; i < 12; ++i) a.convs.push_back({kTrunk[i], i >= prelu_from ? kPrelu : kRelu});
    for (int i = 1; i < 12; ++i)
        a.layers.push_back({0, {i}, std::min(kTrunk[i].cout, 128), kPoolAfter[i], kPermNone, kTrunkWiring[i - 1], -1});
    memcpy(a.act_c, kActC, sizeof(kActC));
    a.zero_pads[CAT] = true;
    return a;
}

// rtpose (rtpose_vgg.py:69-127): state_dict order is the trunk, then branch 0 (PAF) stages 1 .. 6, then branch 1
// (heat map) stages 1 .. 6.  Each layer of a stage runs both branches as one two-group launch.
NetArch rtpose_arch() {
    NetArch a = trunk_arch(12);
    a.name = "rtpose";
    a.stages = kStages;
    int first[2][kStages + 1];      // conv of layer 0 of branch b, stage s
    for (int b = 0; b < 2; ++b)
        for (int s = 1; s <= kStages; ++s) {
            const int outc = b == 0 ? kPaf : kHeat;
            const std::vector<ConvSpec> convs = s == 1
                ? std::vector<ConvSpec>{{128, 128, 3}, {128, 128, 3}, {128, 128, 3}, {128, 512, 1}, {512, outc, 1}}
                : std::vector<ConvSpec>{{kCat, 128, 7}, {128, 128, 7}, {128, 128, 7}, {128, 128, 7}, {128, 128, 7},
                                        {128, 128, 1}, {128, outc, 1}};
            first[b][s] = (int)a.convs.size();
            for (const ConvSpec& c : convs) a.convs.push_back({c, kRelu});
            a.convs.back().act = kNoAct;      // the head
        }
    for (int s = 1; s <= kStages; ++s)
        for (int li = 0; li < (s == 1 ? 5 : 7); ++li) {
            const Wiring& wr = (s == 1 ? kStage1Wiring : kStageWiring)[li];
            a.layers.push_back({s, {first[0][s] + li, first[1][s] + li}, wr.maps ? 48 : 128, 0,
                                s > 1 && li == 0 ? kPermRtposeCat : kPermNone, wr, wr.maps ? 2 * (s - 1) : -1});
        }
    for (int i = 0; i < 12; ++i) a.map_ch[i] = i % 2 == 0 ? kPaf : kHeat;
    for (int k = 1; k <= kStages; ++k) a.out[k] = {2 * k, 2 * k - 2, 2 * k - 1};
    return a;
}

// OpenPose_Model(l2, l1): state_dict order is the trunk, then 17 convs per stage (Mconv1_0 .. Mconv5_2, Mconv6, Mconv7),
// one launch each; stage t writes map t.  n-tiles: 48 for the 96-channel convs (two tiles, no pad lanes), 128 for the
// others; the heads 64 (PAF: zero rows 38..63 store +0 over the heat slot) and 32 (heat map).
// DESIGN §2.11: bra and brb hold 768 channels, six 128-channel slots: a dense block's three outputs go to
// slots 0, 1, 2 (stages of 128 inner channels) or 3, 4, 5 (the 96-channel first stage of each branch: lanes 96..127 of
// those slots are never written and stay +0).  Blocks 1, 3, 5 write bra, blocks 2, 4 brb: Mconv{b}_0 reads all three
// slots of the other buffer, _1 reads slot 0 and writes slot 1, _2 reads slot 1 and writes slot 2.  Mconv6 writes br512
// (512 channels).  The PAF heads store 64 lanes at channel 0 of the concat buffer - PAF, then +0 from zero rows and bias
// over the heat slot and the pad lanes, so that an L2 stage >= 2 or L1 stage 1, which reads the heat slot against zero
// weights, never reads an earlier forward's values; the heat-map heads store the 24 lanes from channel 40.
NetArch openpose_arch(int l2, int l1) {
    NetArch a = trunk_arch(9);
    a.name = "OpenPose_Model(" + std::to_string(l2) + ", " + std::to_string(l1) + ")";
    a.l2 = l2;
    a.l1 = l1;
    a.stages = l2 + l1;
    auto add = [&](ConvSpec s, Nonlin act, ArchLayer l) {      // a conv and its launch
        l.convs = {(int)a.convs.size()};
        a.convs.push_back({s, act});
        a.layers.push_back(l);
    };
    for (int t = 0; t < l2 + l1; ++t) {
        const OpStage g = op_stage(l2, t);
        const int base = g.first ? 384 : 0, n = g.inner == 96 ? 48 : 128;     // first slot; n-tile and lanes stored
        for (int b = 0; b < 5; ++b) {      // Mconv{b + 1}_{0,1,2}
            const int cur = b % 2 ? BRB : BRA, prev = b % 2 ? BRA : BRB;
            if (b == 0)
                add({g.in, g.inner, 3}, kPrelu, {t + 1, {}, n, 0, t == 0 ? kPermNone : (g.paf || g.first ? kPermFeatPaf : kPermFeatHeatPaf),
                                                 {CAT, t == 0 ? 64 : 0, 0, cur, {base, 0}, {n, 0}}, -1});
            else
                add({3 * g.inner, g.inner, 3}, kPrelu, {t + 1, {}, n, 0, kPermSlots, {prev, base, 0, cur, {base, 0}, {n, 0}}, -1});
            for (int j = 1; j < 3; ++j)
                add({g.inner, g.inner, 3}, kPrelu,
                    {t + 1, {}, n, 0, kPermNone, {cur, base + 128 * (j - 1), 0, cur, {base + 128 * j, 0}, {n, 0}}, -1});
        }
        add({3 * g.inner, g.innerout, 1}, kPrelu, {t + 1, {}, 128, 0, kPermSlots, {BRA, base, 0, BR512, {0, 0}, {128, 0}}, -1});
        add({g.innerout, g.out, 1}, kNoAct,
            {t + 1, {}, g.paf ? 64 : 32, 0, kPermNone, {BR512, 0, 0, CAT, {g.paf ? 0 : 40, 0}, {g.paf ? 64 : 24, 0}, true}, t});
    }
    a.act_c[BRA] = a.act_c[BRB] = 768;
    a.act_c[BR512] = 512;
    a.zero_pads[BRA] = a.zero_pads[BRB] = true;     // the 96-channel dense-block slots
    for (int i = 0; i < 12; ++i) a.map_ch[i] = i < l2 ? kPaf : kHeat;
    a.out[l2 + l1] = {l2 + l1, l2 - 1, l2 + l1 - 1};
    return a;
}

// state_dict tensor `index` of architecture a: conv *ci, *kind 0 = weight, 1 = bias, 2 = PReLU slope.  False when out of
// range.
bool arch_tensor(const NetArch& a, int index, int* ci, int* kind) {
    if (index < 0) return false;
    for (int c = 0; c < (int)a.convs.size(); ++c) {
        const int nt = a.convs[c].act == kPrelu ? 3 : 2;
        if (index < nt) {
            *ci = c;
            *kind = index;
            return true;
        }
        index -= nt;
    }
    return false;
}
int arch_num_tensors(const NetArch& a) {
    int n = 0;
    for (const ArchConv& c : a.convs) n += c.act == kPrelu ? 3 : 2;
    return n;
}
int arch_tensor_shape(const NetArch& a, int index, long dims[4]) {
    int ci, kind;
    if (!arch_tensor(a, index, &ci, &kind)) return -1;
    const ConvSpec s = a.convs[ci].s;
    dims[0] = s.cout;
    if (kind != 0) return 1;
    dims[1] = s.cin; dims[2] = s.ks; dims[3] = s.ks;
    return 4;
}

struct PlanLaunch {
    ConvTcArgs a;
    double flops;          // algorithmic (unpadded) FLOPs
    int in, out;           // activation buffers (Act); ConvTcArgs keeps only tensor maps of the input
    int f32[2];            // fp32 stage map written per group, -1 = none
};

// Device addresses a plan's tensor maps and arguments point into: activation buffers, residual planes, stage maps.
using PlanBuffers = std::array<const void*, 2 * kNumAct + 12 + 2>;    // + the format's aux table, the fp8 exponent table

// The launch list of one (n, H, W, format, stages) key, valid while `buffers` are still the net's: the trunk and the
// launches of stages 1 .. stages.
struct Plan {
    int n, H, W;
    TcFormat fmt;
    int stages;
    std::vector<PlanLaunch> launches;
    PlanBuffers buffers;
};

// What the last successful forward ran; b200pose_net_last_maps, _profile and the _debug_* hooks read it.
struct LastForward {
    int n = 0, H = 0, W = 0;
    bool fp32 = false;           // the fp32 path ran, else the tensor-core path in format fmt
    TcFormat fmt = TcFormat::kBf16;
    int stages = kStages;        // stages run; the final maps are stage `stages`'s (out_f32[2 stages - 2], [2 stages - 1])
    const void* in = nullptr;    // device input
    int in_u8 = 0;               // normalisation of a uint8 input fused into conv1_1 (0: fp32 input)
    const int* ext = nullptr;    // extents table of a ragged forward, null: uniform
    std::vector<int> ext_host;   // ... and its host copy {H_0, W_0, ...} (empty: uniform)
};

}  // namespace

struct b200pose_net {
    int device = 0, num_sms = 0;
    // architecture, fixed at creation: rtpose, or OpenPose_Model(l2, l1) (b200pose_net_create_openpose)
    NetArch arch;
    bool finalized = false;
    std::vector<std::vector<float>> host_w, host_b, host_slope;   // per conv (slope: PReLU convs only)
    std::vector<bool> have;                                        // per tensor
    std::vector<DevBuf<float>> d_w, d_b, d_slope;      // per conv, fp32 OIHW (parity mode, conv1_1) and PReLU slopes
    std::vector<TcLayer> tc;                           // per layer of arch
    // Plans of the last 32 keys are kept, so that alternating shapes (multi-scale, mixed frame sizes) do not re-encode
    // up to 51 tensor maps and synchronise the stream.  `plan` is the one the last tensor-core forward selected.
    std::list<Plan> plans;
    const Plan* plan = nullptr;
    // The launches of a forward pass (52 with six stages) are captured at the second use of a (shape, format, stages,
    // input pointer) into a CUDA graph and replayed (B200POSE_GRAPH=0: plain launches).  Graphs embed the tensor maps,
    // i.e. buffer addresses: every plan build drops them.  Capture needs a real stream: calls on the legacy default stream
    // (0) launch directly.
    using GraphKey = std::tuple<int, int, int, TcFormat, int, int, bool, const void*>;   // n, H, W, format, stages, in_u8, ragged, input
    bool use_graph = true;
    std::map<GraphKey, GraphExec> graphs;
    std::set<GraphKey> graph_seen;    // a key is captured at its SECOND use: callers that pass a fresh pointer every time never pay a capture
    // bf16 (fp16: binary16) activation buffers by Act id, and their residual ("lo") planes (bf16x3 only)
    DevBuf<__nv_bfloat16> act[kNumAct], act_lo[kNumAct];
    DevBuf<float> in_stage, out_f32[12];
    // fp32 parity buffers
    DevBuf<float> f_a, f_b, f_cat, f_x, f_y, f_in, f_u8;
    DevBuf<float> f_cat3, f_z;         // OpenPose_Model: cat[features, heat, paf], Mconv6's output
    LastForward last;
    DevBuf<unsigned char> in_stage_u8;
    int preprocess = 1;                // normalisation fused into the uint8 entry points (preprocess_core.h; 1 = rtpose)
    int stages = kStages;              // refinement stages every later forward runs (b200pose_net_set_stages)
    bool jpeg_progressive = false;     // the JPEG calls decode progressive streams (b200pose_net_set_jpeg_progressive)
    DevBuf<unsigned char> raw_stage;   // raw (un-resized) frames of b200pose_*crop* / b200pose_infer_raw_u8
    // Ragged batches (DESIGN.md §1): the extents table [H_0, W_0, H_1, W_1, ...] every kernel of a ragged forward reads.
    // Allocated once for kMaxRagged images and never moved, so that plans and captured graphs stay valid across mixes;
    // rewritten on the stream before each ragged forward.
    DevBuf<int> d_ext;
    std::vector<int> ext_host;     // what upload_ext last wrote into d_ext
    DevBuf<RaggedFrame> d_frames;      // frame table (per-frame source geometry) of the last crop or uint8 mirror
    // video frames (b200pose_net_convert_frames, b200pose_infer_frames): the planes of host frames, packed, and the
    // source table of the last conversion
    DevBuf<unsigned char> frame_stage;
    DevBuf<FrameSrc> d_frame_src;
    // JPEG streams (b200pose_net_decode_jpegs, b200pose_infer_jpegs): the call's upload (descriptors, segment and chunk
    // tables, status words, scan bytes), the unstuffed scans, the coefficients and the sample planes
    DevBuf<char> jpeg_in;
    DevBuf<unsigned char> jpeg_data, jpeg_planes;
    DevBuf<short> jpeg_coef;
    // JPEG encoding (b200pose_net_encode_jpegs): the call's upload (descriptors, Huffman tables) followed by the per-image
    // bit counts and stream sizes, staged host frames, the coefficients, per-block code lengths and bit offsets, the
    // bit buffers, and the streams of a call whose output is on the host
    DevBuf<char> jenc_in;
    DevBuf<unsigned char> jenc_frames, jenc_out;
    DevBuf<short> jenc_coef;
    DevBuf<int> jenc_acbits;
    DevBuf<long long> jenc_off;
    DevBuf<unsigned> jenc_words;
    // PNG encoding (b200pose_net_encode_pngs): the call's upload (descriptors, per-image results, deflate word offsets),
    // staged host frames, the filtered bytes, the tile table, the symbols, the blocks, the deflate words, and the files
    // of a call whose output is on the host
    DevBuf<char> penc_in;
    DevBuf<unsigned char> penc_frames, penc_filt, penc_out;
    DevBuf<long long> penc_tiles;
    DevBuf<unsigned short> penc_sym;
    DevBuf<PngBlock> penc_blocks;
    DevBuf<unsigned> penc_words;
    // PNG streams (b200pose_net_decode_pngs, b200pose_infer_pngs): the call's upload (descriptors, IDAT table, status
    // words, IDAT chunks), the gathered zlib streams and the inflated rows
    DevBuf<char> png_in;
    DevBuf<unsigned char> png_zlib, png_rows;
    // training batches (b200pose_net_augment): the sample table and L sums, staged host frames, the horizontal passes,
    // the jittered images, the images of the JPEG round trip, and the outputs of a call whose outputs are on the host
    DevBuf<char> aug_in;
    DevBuf<unsigned char> aug_src, aug_tmp, aug_px, aug_jpeg, aug_u8;
    DevBuf<float> aug_out;
    // fp8 mode (DESIGN.md §2.3): amax[launch * n + image] = max |bf16| (fp32 bits) launch (0 = conv1_1) stored for the
    // image; zeroed at the start of every fp8 forward
    DevBuf<unsigned> amax;
    DevBuf<int> ea;                    // ea[launch * n + image]: the activation exponent the fp8 kernel used
    // fp16 mode: ovf[image] = 1 when a launch stored a value beyond binary16's range for the image; zeroed at the start
    // of every fp16 forward
    DevBuf<unsigned> ovf;
    ~b200pose_net() { graphs.clear(); }     // the graph execs go before the buffers they point into
};

struct b200pose_post {
    int device = 0;
    PostBuffers pb{};
    DevBuf<float> d_heat, d_paf;
    DevBuf<float> tta_in, tta_out;   // b200pose_flip_merge staging for host pointers
    // Results are copied to pinned host memory by the run itself (second stream, right after the assembly) into one
    // of two slots selected by the run's parity, so the host can fetch run i while run i+1 is in flight.
    Stream s2;
    Event ev_limbs, ev_asm, ev_fetch[2];
    long runs = 0;                  // runs submitted so far; ticket of the latest = runs - 1
    int slot_n[2] = {0, 0};
    HostBuf<int> hp_nh[2], hp_status[2], hp_counts[2];
    HostBuf<float> hp_humans[2];
    int cur = 0;                    // slot the getters read
    long cur_ticket = -1;
    std::vector<float> h_px_s;
    std::vector<int> h_px, h_py;
    int hw_h = 0, hw_w = 0;
    // Peaks / limbs / assembly of run i all run on the second stream from a private copy of the maps (15 MB at batch 32),
    // so that the caller's stream is free for the convolutions of run i+1: the small kernels (peaks, assembly) co-reside
    // with the conv CTAs and the limbs blocks fill the SMs the conv launches leave idle in their last wave.
    DevBuf<float> ov_maps[2];                      // [heat | paf] copies, slot = run parity
    Event ev_maps, ev_ld[2];                       // maps copied (st) / limbs done with a slot (s2)
    bool have_ld[2] = {false, false};
    // extents of a ragged run, slot = run parity: the peaks / limbs of run i on the second stream still read them while
    // run i+1 rewrites the net's table
    DevBuf<int> d_ext[2];
    // ragged multi-scale averaging: the frames' base extents (the net's table holds the last scale's) and the resize
    // geometry of every (scale, frame)
    DevBuf<int> ms_ext;
    DevBuf<RaggedResize> ms_resize;
    // fp16 overflow flags of the fused runs, slot = run parity: one row of 2 * batch_cap images per forward of the run (a
    // multi-scale run makes one forward per scale), copied from the net's flags behind each forward
    HostBuf<unsigned> hp_ovf[2];
    // b200pose_post_draw: the call's images, person rows and frame table (copied from pageable memory, so a later run
    // may reuse the pinned slot at once), its planned primitives, host frames' staging; ev_draw: the last draw is done
    DevBuf<char> draw_job;
    DevBuf<DrawPrim> draw_prims;
    DevBuf<unsigned char> draw_frames;
    Event ev_draw;
    bool have_draw = false;
    int ovf_rows[2] = {0, 0}, ovf_imgs[2] = {0, 0};    // forwards copied, images per forward (2n with flip)
    int ovf_pending = 0, ovf_pending_imgs = 0;          // ... of the run being enqueued
    // JPEG status words of a run made from JPEG streams, slot = run parity; jpeg_imgs: images copied (0: another run)
    HostBuf<unsigned> hp_jpeg[2];
    int jpeg_imgs[2] = {0, 0}, jpeg_pending = 0;
    // the same for a run made from PNG streams
    HostBuf<unsigned> hp_png[2];
    int png_imgs[2] = {0, 0}, png_pending = 0;
    // scoring / prune settings of the runs submitted from now on (b200pose_post_set_params); they travel to the kernels
    // by value, so a run in flight keeps its own
    PostParams params{DefaultPostParams::paf_thresh, DefaultPostParams::paf_samples, DefaultPostParams::paf_min_above,
                      DefaultPostParams::min_parts, DefaultPostParams::min_person_score};
    // grids of limb_score_kernel / range_sort_kernel for the runs submitted from now on, 0 = the defaults
    // (b200pose_post_set_grids, a test hook: the results never depend on them)
    int score_blocks = 0, sort_blocks = 0;
    // peak refinement of the runs submitted from now on (b200pose_post_set_refine), passed to the kernels by value
    int refine = B200POSE_REFINE_CUBIC;
    // the second stream's work still reads the buffers; post_free is null-safe (post_alloc zeroes pb first)
    ~b200pose_post() { if (s2) cudaStreamSynchronize(s2); post_free(pb); }
};

namespace {

bool is_openpose(const b200pose_net* net) { return net->arch.l2 > 0; }

// The final maps of the last forward: the PAF and heatmap of its last stage (OpenPose_Model: of its last L2 and L1
// stages).
const float* last_paf(const b200pose_net* net) { return net->out_f32[net->arch.out[net->last.stages].paf].p; }
const float* last_heat(const b200pose_net* net) { return net->out_f32[net->arch.out[net->last.stages].heat].p; }

// Calls row(g, o, r, w) for output channel o of every group g of layer L (packed row r = g * cout_pad + o), w its fp32
// weights in packed order [tap][cin_pad]: input channels at their physical channel of the buffer the layer reads
// (perm_phys), zero in the pad channels.
template <class F> void for_each_weight_row(const b200pose_net* net, const TcLayer& L, F&& row) {
    const int taps = L.ks * L.ks, cin_pad = L.cin_blocks * 64, cout_pad = L.n_tiles * L.n_tile;
    std::vector<float> w((size_t)taps * cin_pad);
    for (int g = 0; g < L.groups; ++g) {
        const ConvSpec s = net->arch.convs[L.convs[g]].s;
        const std::vector<float>& hw = net->host_w[L.convs[g]];
        for (int o = 0; o < s.cout; ++o) {
            std::fill(w.begin(), w.end(), 0.f);
            for (int c = 0; c < s.cin; ++c)
                for (int t = 0; t < taps; ++t)
                    w[(size_t)t * cin_pad + perm_phys(L.perm, L.slot, c)] = hw[((size_t)o * s.cin + c) * taps + t];
            row(g, o, g * cout_pad + o, w.data());
        }
    }
}

// The tensor-core layer of arch layer l, before any weights are packed.  Its input is 192 channels of the concat buffer
// (the concat permutations), three 128-channel slots (kPermSlots) or the conv's input channels rounded up to 64.
TcLayer make_tc_layer(const NetArch& arch, const ArchLayer& l) {
    const ArchConv& c0 = arch.convs[l.convs[0]];
    const ConvSpec sp = c0.s;
    const int cin_pad = l.perm == kPermSlots ? 3 * 128 : (l.perm != kPermNone ? 192 : (sp.cin + 63) / 64 * 64);
    const int cout_pad = ((sp.cout + l.n_tile - 1) / l.n_tile) * l.n_tile;
    TcLayer L;
    L.ks = sp.ks; L.cin_blocks = cin_pad / 64; L.groups = (int)l.convs.size(); L.n_tile = l.n_tile; L.n_tiles = cout_pad / l.n_tile;
    L.relu = c0.act == kRelu; L.pool = l.pool; L.prelu = c0.act == kPrelu; L.convs = l.convs; L.perm = l.perm; L.slot = sp.cin / 3;
    for (int c : l.convs) L.macs_per_pixel += (double)arch.convs[c].s.cin * arch.convs[c].s.cout * sp.ks * sp.ks;
    return L;
}

// bf16 weights of layer L and its bias (every format's): [hi taps | lo taps], bf16(w) and the residual bf16(w - hi) (read
// by bf16x3 only)
int pack_tc_layer(b200pose_net* net, TcLayer& L) {
    const int taps = L.ks * L.ks, cin_pad = L.cin_blocks * 64, rows = L.groups * L.n_tiles * L.n_tile;
    std::vector<uint16_t> w((size_t)2 * taps * rows * cin_pad, 0);
    std::vector<float> b((size_t)rows, 0.f), s(L.prelu ? rows : 0, 0.f);
    for_each_weight_row(net, L, [&](int g, int o, int r, const float* wr) {
        b[r] = net->host_b[L.convs[g]][o];
        if (L.prelu) s[r] = net->host_slope[L.convs[g]][o];
        for (int t = 0; t < taps; ++t)
            for (int k = 0; k < cin_pad; ++k) {
                const float wf = wr[(size_t)t * cin_pad + k];
                const uint16_t hi = f2bf(wf);
                w[((size_t)t * rows + r) * cin_pad + k] = hi;
                w[((size_t)(taps + t) * rows + r) * cin_pad + k] = f2bf(wf - bf2f(hi));
            }
    });
    DevBuf<unsigned char>& dw = L.w[(int)TcWeights::kBf16HiLo];
    CU(dw.ensure(w.size() * 2));
    CU(L.bias.ensure(b.size()));
    CU(cudaMemcpy(dw.p, w.data(), w.size() * 2, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(L.bias.p, b.data(), b.size() * 4, cudaMemcpyHostToDevice));
    if (L.prelu) {
        CU(L.slope.ensure(s.size()));
        CU(cudaMemcpy(L.slope.p, s.data(), s.size() * 4, cudaMemcpyHostToDevice));
    }
    return 0;
}

// fp8 weights of layer L (half the bytes of the bf16 ones): per output row ew = floor(log2(448 / max|w_row|)) and
// e4m3(w * 2^ew), one rounding from the fp32 weight; each 32-channel slice in the K order the kernel's A fragments have
// (fp8_k_to_channel).
int pack_fp8_layer(const b200pose_net* net, TcLayer& L) {
    const int taps = L.ks * L.ks, cin_pad = L.cin_blocks * 64, rows = L.groups * L.n_tiles * L.n_tile;
    L.h_w_exp.assign(rows, 0);
    std::vector<uint8_t> w8((size_t)taps * rows * cin_pad, 0);
    for_each_weight_row(net, L, [&](int, int, int r, const float* wr) {
        float m = 0.f;
        for (size_t i = 0; i < (size_t)taps * cin_pad; ++i) m = std::max(m, std::fabs(wr[i]));
        uint32_t mb;
        memcpy(&mb, &m, 4);
        const int ew = fp8_exp_from_amax(mb);
        L.h_w_exp[r] = ew;
        for (int t = 0; t < taps; ++t) {
            const float* src = wr + (size_t)t * cin_pad;
            uint8_t* dst = &w8[((size_t)t * rows + r) * cin_pad];
            for (int k = 0; k < cin_pad; ++k) dst[k] = e4m3_rn_bits(src[(k & ~31) + fp8_k_to_channel(k & 31)] * exp2_int(ew));
        }
    });
    DevBuf<unsigned char>& dw = L.w[(int)TcWeights::kE4m3];
    CU(dw.ensure(w8.size()));
    CU(L.w_exp.ensure(rows));
    CU(cudaMemcpy(dw.p, w8.data(), w8.size(), cudaMemcpyHostToDevice));
    CU(cudaMemcpy(L.w_exp.p, L.h_w_exp.data(), rows * sizeof(int), cudaMemcpyHostToDevice));
    return 0;
}

// fp16 mode: a weight beyond binary16's range would be +-inf, and inf * 0 = NaN sums can be turned into a finite 0 by
// the ReLU, i.e. not reported by the overflow flags; such weights are refused instead.
int check_f16_weight(float w, int conv) {
    const uint16_t h = f16_rn_bits(w);
    if ((h & 0x7c00u) == 0x7c00u) return fail("fp16 mode: conv %d has weight %g, beyond binary16's range (65504)", conv, w);
    return 0;
}

// fp16 weights of layer L: binary16(w), one rounding from the fp32 weight, in the layout of the bf16 value slices (pad
// rows and channels 0).
int pack_f16_layer(const b200pose_net* net, TcLayer& L) {
    const int taps = L.ks * L.ks, cin_pad = L.cin_blocks * 64, rows = L.groups * L.n_tiles * L.n_tile;
    std::vector<uint16_t> w16((size_t)taps * rows * cin_pad, 0);
    int rc = 0;
    for_each_weight_row(net, L, [&](int g, int, int r, const float* wr) {
        for (int t = 0; t < taps; ++t)
            for (int k = 0; k < cin_pad; ++k) {
                const float w = wr[(size_t)t * cin_pad + k];
                if (rc == 0) rc = check_f16_weight(w, L.convs[g]);
                w16[((size_t)t * rows + r) * cin_pad + k] = f16_rn_bits(w);
            }
    });
    if (rc) return rc;
    DevBuf<unsigned char>& dw = L.w[(int)TcWeights::kBinary16];
    CU(dw.ensure(w16.size() * 2));
    CU(cudaMemcpy(dw.p, w16.data(), w16.size() * 2, cudaMemcpyHostToDevice));
    return 0;
}

// Packs the weights of layer L that format fmt reads, unless they are packed already.  The bf16 ones (with the bias) are
// packed at finalize, the e4m3 and binary16 ones when the first plan of their format is built: nets that never run those
// formats do not pay for them.
int ensure_packed(b200pose_net* net, TcLayer& L, TcFormat fmt) {
    const TcWeights enc = tc_weights(fmt);
    if (L.w[(int)enc].p != nullptr) return 0;
    int rc;
    switch (enc) {
        case TcWeights::kBf16HiLo: rc = pack_tc_layer(net, L); break;
        case TcWeights::kE4m3: rc = pack_fp8_layer(net, L); break;
        case TcWeights::kBinary16: rc = pack_f16_layer(net, L); break;
        default: return fail("unknown weight encoding %d", (int)enc);
    }
    if (rc) L.w[(int)enc].release();      // a pack that failed part-way is redone by the next call
    return rc;
}

// The per-image table of format f (tc_aux): fp8 amax rows (conv1_1, then each launch), fp16 overflow flags; null otherwise.
unsigned* aux_table(const b200pose_net* net, TcFormat f) {
    switch (tc_aux(f)) {
        case TcAux::kAmax: return net->amax.p;
        case TcAux::kOverflow: return net->ovf.p;
        case TcAux::kNone: break;
    }
    return nullptr;
}

// Small-batch plans: the 46 x 46 stage layers (two groups) would fill at most half of the SMs with one n-tile per group.
// Their launches are the launch-bound part of the product: they are chained by PDL and replayed as a CUDA graph; the large
// plans are GPU-bound and get neither (a capture only adds a CPU hiccup).
bool small_plan(const b200pose_net* net, int n, int H, int W) {
    return 2 * n * ((H / 8 + kTileH - 1) / kTileH) * ((W / 8 + kTileW - 1) / kTileW) * 2 <= net->num_sms;
}

// Appends tensor-core layer L, wired as `wr`, to plan p; a stage head writes the fp32 maps map0 (group 0) and map0 + 1
// (group 1).  fp8: writers[] are the launches (amax table rows) that wrote the channels it reads; writers[1] may be -1.
int add_plan(const b200pose_net* net, Plan& p, const TcLayer& L, const Wiring& wr, int map0, const int writers[2]) {
    const int n = p.n, H = p.H / kActDiv[wr.in], W = p.W / kActDiv[wr.in];
    ConvTcArgs a;
    memset(&a, 0, sizeof(a));
    a.fmt = p.fmt;
    a.n_img = n; a.H = H; a.W = W; a.ksize = L.ks; a.cin_blocks = L.cin_blocks;
    a.in_ch_base = wr.in_base; a.in_ch_group_stride = wr.in_group_stride; a.groups = L.groups;
    a.n_tile = L.n_tile; a.n_tiles = L.n_tiles; a.bias = L.bias.p; a.relu = L.relu; a.pool = L.pool;
    a.slope = L.prelu ? L.slope.p : nullptr;
    {   // small batches: while the layer's CTAs fill at most half of the SMs, halve the work per CTA - 128-wide n-tiles become
        // 64-wide, then 32-wide (the weight layout does not depend on the n-tile)
        const int pix = n * ((H + kTileH - 1) / kTileH) * ((W + kTileW - 1) / kTileW);
        if (L.n_tile == 128 && 2 * pix * L.groups * a.n_tiles <= net->num_sms) { a.n_tile = 64; a.n_tiles = L.n_tiles * 2; }
        if (a.n_tile == 64 && 2 * pix * L.groups * a.n_tiles <= net->num_sms) { a.n_tile = 32; a.n_tiles *= 2; }
    }
    const int max_n = tc_max_n_tile(p.fmt);
    if (a.n_tile > max_n) { a.n_tile = max_n; a.n_tiles = L.n_tiles * (L.n_tile / max_n); }
    if (tc_aux(p.fmt) == TcAux::kAmax) {
        const int slot = 1 + (int)p.launches.size();      // amax table row of this launch (0 = conv1_1)
        a.amax_out = net->amax.p + (size_t)slot * n;
        a.amax_in[0] = net->amax.p + (size_t)writers[0] * n;
        a.amax_in[1] = writers[1] >= 0 ? net->amax.p + (size_t)writers[1] * n : nullptr;
        a.w_exp = L.w_exp.p;
        a.ea_out = net->ea.p + (size_t)slot * n;
    }
    if (tc_aux(p.fmt) == TcAux::kOverflow) a.ovf_out = net->ovf.p;
    a.out = net->act[wr.out].p; a.out_cstride = net->arch.act_c[wr.out];
    a.out_ch_off[0] = wr.out_off[0]; a.out_ch_off[1] = wr.out_off[1];
    a.store_ch[0] = wr.store[0]; a.store_ch[1] = wr.store[1];
    const int f32[2] = {wr.maps ? map0 : -1, wr.maps && L.groups == 2 ? map0 + 1 : -1};
    for (int g = 0; g < 2; ++g)
        if (f32[g] >= 0) {
            a.out_f32[g] = net->out_f32[f32[g]].p;
            a.f32_ch[g] = net->arch.map_ch[f32[g]];
        }
    // small batches (the 46 x 46 layers fill less than half of the SMs with 16 x 16 tiles): chain the layers with programmatic
    // dependent launches; the first tensor-core layer follows conv1_1, which does not signal.  small_plan gets this
    // layer's H, W and divides them by 8 again (DESIGN §2.1).
    a.pdl = (!p.launches.empty() && small_plan(net, n, H, W)) ? 1 : 0;
    while ((a.H << a.ext_shift) < p.H) ++a.ext_shift;      // ragged batches: the launch's output resolution relative to the input
    a.ext_shift += a.pool;
    const __nv_bfloat16* in_lo = nullptr;
    if (tc_planes(p.fmt) == 2) {
        in_lo = net->act_lo[wr.in].p;
        a.out_lo = net->act_lo[wr.out].p;
    }
    cudaError_t e = conv_tc_make_maps(a, net->act[wr.in].p, net->arch.act_c[wr.in], L.w[(int)tc_weights(p.fmt)].p, in_lo);
    if (e != cudaSuccess) return cuda_fail("conv_tc_make_maps failed: %s", cudaGetErrorString(e));
    p.launches.push_back({a, 2.0 * n * H * W * L.macs_per_pixel, wr.in, wr.out, {f32[0], f32[1]}});
    return 0;
}

// fp8 plans also point into the amax and exponent tables, fp16 plans into the overflow flags (only plans of that format
// do, so only they depend on them)
PlanBuffers plan_buffers(const b200pose_net* net, TcFormat fmt) {
    PlanBuffers b;
    for (int i = 0; i < kNumAct; ++i) {
        b[i] = net->act[i].p;
        b[kNumAct + i] = net->act_lo[i].p;
    }
    for (int i = 0; i < 12; ++i) b[2 * kNumAct + i] = net->out_f32[i].p;
    b[2 * kNumAct + 12] = aux_table(net, fmt);
    b[2 * kNumAct + 13] = tc_aux(fmt) == TcAux::kAmax ? net->ea.p : nullptr;
    return b;
}

// Fills p.launches, (re)allocating the buffers of p's key.
int build_plan_tc(b200pose_net* net, Plan& p, cudaStream_t st) {
    const size_t px = (size_t)p.n * p.H * p.W;
    for (int plane = 0; plane < tc_planes(p.fmt); ++plane) {
        DevBuf<__nv_bfloat16>* bufs = plane ? net->act_lo : net->act;
        for (int i = 0; i < kNumAct; ++i) CU(bufs[i].ensure(px / (kActDiv[i] * kActDiv[i]) * net->arch.act_c[i]));
        // pad lanes no launch writes must read as zero; on the caller's stream (a non-blocking stream is not ordered
        // against the legacy default stream a plain cudaMemset would use)
        for (int i = 0; i < kNumAct; ++i)
            if (net->arch.zero_pads[i])
                CU(cudaMemsetAsync(bufs[i].p, 0, px / (kActDiv[i] * kActDiv[i]) * net->arch.act_c[i] * 2, st));
    }
    for (int i = 0; i < 12; ++i) CU(net->out_f32[i].ensure(px / 64 * net->arch.map_ch[i]));
    if (tc_aux(p.fmt) == TcAux::kAmax) {     // rows for every layer whatever p.stages: plans of every stage count share them
        const size_t rows = 1 + net->arch.layers.size();
        CU(net->amax.ensure(rows * p.n));
        CU(net->ea.ensure(rows * p.n));
    }
    if (tc_aux(p.fmt) == TcAux::kOverflow) CU(net->ovf.ensure((size_t)p.n));
    if (tc_binary16(p.fmt))
        for (float w : net->host_w[0])      // conv1_1 converts its fp32 weights in the kernel
            if (check_f16_weight(w, 0)) return 1;
    for (TcLayer& L : net->tc)
        if (ensure_packed(net, L, p.fmt)) return 1;
    // fp8: the launch that last wrote each buffer (amax table row); the concat buffer has two writers, conv4_4_CPM
    // (features) and the latest stage head (PAF + heatmap)
    int writer[kNumAct], cat_head = -1;
    for (int& w : writer) w = -1;
    writer[T1] = 0;
    for (size_t k = 0; k < net->tc.size() && net->arch.layers[k].stage <= p.stages; ++k) {
        const Wiring& wr = net->arch.layers[k].wiring;
        const int ws[2] = {writer[wr.in], wr.in == CAT && wr.in_base == 0 ? cat_head : -1};
        if (add_plan(net, p, net->tc[k], wr, net->arch.layers[k].map0, ws)) return 1;
        if (wr.out == CAT && wr.maps) cat_head = (int)p.launches.size();
        else writer[wr.out] = (int)p.launches.size();
    }
    p.buffers = plan_buffers(net, p.fmt);
    return 0;
}

void drop_graphs(b200pose_net* net) {
    net->graphs.clear();
    net->graph_seen.clear();
}

// Points net->plan at the plan of (n, H, W, fmt, stages): a kept one whose buffers are still the net's, or a new one
// (the oldest of 32 is dropped).  A build may move the buffers the captured graphs point into: it synchronises the
// stream and drops the graphs first.
int select_plan(b200pose_net* net, int n, int H, int W, TcFormat fmt, int stages, cudaStream_t st) {
    const PlanBuffers bufs = plan_buffers(net, fmt);
    auto same_key = [&](const Plan& p) { return p.n == n && p.H == H && p.W == W && p.fmt == fmt && p.stages == stages; };
    for (const Plan& p : net->plans)
        if (same_key(p) && p.buffers == bufs) {
            net->plan = &p;
            return 0;
        }
    CU(cudaStreamSynchronize(st));
    drop_graphs(net);
    net->plan = nullptr;
    net->plans.remove_if(same_key);
    if (net->plans.size() >= 32) net->plans.pop_front();
    net->plans.push_back(Plan{n, H, W, fmt, stages, {}, {}});
    if (build_plan_tc(net, net->plans.back(), st)) {
        net->plans.pop_back();
        return 1;
    }
    net->plan = &net->plans.back();
    return 0;
}

// The first k launches of a forward with net->plan: conv1_1, then the plan's.  A ragged forward passes its extents
// table (the plans are shared with uniform batches of the canvas size).  fp8 / fp16: zero_aux clears the format's aux
// table - the amax rows / the overflow flags - first (a memset, not a launch); re-runs of launches (debug_run, profile)
// leave it as it is - they record the same maxima and flags again.
// after (b200pose_net_profile): after[i] is recorded behind launch i.
int launch_forward_tc(const b200pose_net* net, const void* d_in, int in_u8, const int* ext, int k, cudaStream_t st,
                      bool zero_aux = false, const Event* after = nullptr) {
    const Plan& p = *net->plan;
    unsigned* aux = aux_table(net, p.fmt);
    if (aux != nullptr && zero_aux) {
        const size_t rows = tc_aux(p.fmt) == TcAux::kAmax ? 1 + p.launches.size() : 1;
        CU(cudaMemsetAsync(aux, 0, rows * p.n * sizeof(unsigned), st));
    }
    if (k >= 1) {
        CU(conv_first_launch(d_in, in_u8, net->d_w[0].p, net->d_b[0].p, p.fmt, net->act[T1].p,
                             tc_planes(p.fmt) == 2 ? net->act_lo[T1].p : nullptr, aux, p.n, p.H, p.W, ext, st));
        if (after) CU(cudaEventRecord(after[0], st));
    }
    for (int i = 0; i + 1 < k; ++i) {
        ConvTcArgs a = p.launches[i].a;
        a.ext = ext;
        CU(conv_tc_launch(a, net->num_sms, st));
        if (after) CU(cudaEventRecord(after[i + 1], st));
    }
    return 0;
}

int forward_tc(b200pose_net* net, const void* d_in, int in_u8, int n, int H, int W, TcFormat fmt, int stages,
               cudaStream_t st, const int* ext) {
    if (select_plan(net, n, H, W, fmt, stages, st)) return 1;
    const int launches = 1 + (int)net->plan->launches.size();
    cudaGraphExec_t exec = nullptr;
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    if (net->use_graph && small_plan(net, n, H, W) && st != nullptr && cudaStreamIsCapturing(st, &cap) == cudaSuccess &&
        cap == cudaStreamCaptureStatusNone) {
        const b200pose_net::GraphKey key{n, H, W, fmt, stages, in_u8, ext != nullptr, d_in};
        auto it = net->graphs.find(key);
        if (it != net->graphs.end()) {
            exec = it->second;
        } else if (net->graph_seen.insert(key).second) {      // first sight: plain launches
            if (net->graph_seen.size() > 4096) net->graph_seen.clear();
        } else {
            if (net->graphs.size() >= 64) drop_graphs(net);
            cudaGraph_t graph = nullptr;
            CU(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
            const int rc = launch_forward_tc(net, d_in, in_u8, ext, launches, st, true);
            cudaError_t e = cudaStreamEndCapture(st, &graph);
            if (rc == 0 && e == cudaSuccess) e = cudaGraphInstantiate(&exec, graph, 0);
            if (graph) cudaGraphDestroy(graph);
            if (rc == 0 && e == cudaSuccess) {
                net->graphs[key].h = exec;
            } else {      // no graph (e.g. a launch attribute the capture refuses): plain launches from now on
                cudaGetLastError();
                fprintf(stderr, "[b200pose] CUDA graph capture of the forward pass failed (%s): launching directly\n",
                        rc ? b200pose_last_error() : cudaGetErrorString(e));
                net->use_graph = false;
                exec = nullptr;
            }
        }
    }
    if (exec) CU(cudaGraphLaunch(exec, st));
    else if (launch_forward_tc(net, d_in, in_u8, ext, launches, st, true)) return 1;
    g_launches += launches;
    return 0;
}

// The convs of group g of stage s's tensor-core layers, in launch order.
std::vector<int> stage_convs(const NetArch& a, int s, int g) {
    std::vector<int> v;
    for (const ArchLayer& l : a.layers)
        if (l.stage == s) v.push_back(l.convs[g]);
    return v;
}

int forward_fp32(b200pose_net* net, const float* d_in, int n, int H, int W, int stages, cudaStream_t st,
                 const int* ext) {
    const size_t px1 = (size_t)n * H * W;
    const int h = H / 8, w = W / 8;
    const size_t px8 = (size_t)n * h * w;
    CU(net->f_in.ensure(px1 * 3));
    CU(net->f_a.ensure(px1 * 64)); CU(net->f_b.ensure(px1 * 64));
    CU(net->f_cat.ensure(px8 * kCat)); CU(net->f_x.ensure(px8 * 512)); CU(net->f_y.ensure(px8 * 512));
    for (int i = 0; i < 12; ++i) CU(net->out_f32[i].ensure(px8 * net->arch.map_ch[i]));
    const NetArch& arch = net->arch;
    const bool op = is_openpose(net);
    if (op) { CU(net->f_cat3.ensure(px8 * kCat)); CU(net->f_z.ensure(px8 * 512)); }
    CU(nchw_to_nhwc_f32_launch(d_in, net->f_in.p, n, 3, H, W, 3, 0, st));
    ++g_launches;
    const float* cur = net->f_in.p;
    int cur_c = 3, ch = H, cw = W;
    float* ping = net->f_a.p;
    float* pong = net->f_b.p;
    auto conv = [&](int ci, const float* in, int in_cs, int in_off, float* out, int out_cs, int out_off, int hh, int ww,
                    float* nchw) -> int {
        const ConvSpec s = arch.convs[ci].s;
        ConvF32Args a;
        a.in = in; a.in_cstride = in_cs; a.in_ch_off = in_off; a.w = net->d_w[ci].p; a.bias = net->d_b[ci].p;
        a.out = out; a.out_cstride = out_cs; a.out_ch_off = out_off; a.out_nchw = nchw;
        a.n_img = n; a.H = hh; a.W = ww; a.cin = s.cin; a.cout = s.cout; a.ks = s.ks; a.relu = arch.convs[ci].act == kRelu;
        a.slope = net->d_slope[ci].p;
        a.ext = ext;
        a.ext_shift = 0;
        while ((hh << a.ext_shift) < H) ++a.ext_shift;
        CU(conv_f32_launch(a, st));
        ++g_launches;
        return 0;
    };
    for (int i = 0; i < 12; ++i) {
        const ConvSpec s = kTrunk[i];
        const bool last = (i == 11);
        float* dst = last ? net->f_cat.p : ping;
        // OpenPose_Model: the features go to cat[features, paf] at channel 0, and through f_z (NCHW) into
        // cat[features, heat, paf]
        const int cat_cs = op ? kFeat + kPaf : kCat, cat_off = op ? 0 : kPaf + kHeat;
        if (conv(i, cur, cur_c, 0, dst, last ? cat_cs : s.cout, last ? cat_off : 0, ch, cw, last && op ? net->f_z.p : nullptr))
            return 1;
        cur = dst; cur_c = s.cout;
        std::swap(ping, pong);
        if (kPoolAfter[i]) {
            CU(maxpool_f32_launch(cur, ping, n, ch, cw, cur_c, st));
            ++g_launches;
            cur = ping; ch /= 2; cw /= 2;
            std::swap(ping, pong);
        }
    }
    if (op) {
        // inputs in the reference's channel order: f_cat = cat[features, paf], f_cat3 = cat[features, heat, paf]; a
        // dense block's three outputs side by side in f_x (blocks 1, 3, 5) or f_y (2, 4); Mconv6 -> f_z; the head's
        // NHWC output is scratch (f_y), its NCHW copy the stage map
        constexpr int kCat2 = kFeat + kPaf, kCat3 = kFeat + kHeat + kPaf;
        CU(nchw_to_nhwc_f32_launch(net->f_z.p, net->f_cat3.p, n, kFeat, h, w, kCat3, 0, st));
        ++g_launches;
        for (int t = 0; t < arch.stages; ++t) {
            const OpStage g = op_stage(arch.l2, t);
            const std::vector<int> ci = stage_convs(arch, t + 1, 0);
            const int cs = 3 * g.inner;
            float* blk[2] = {net->f_x.p, net->f_y.p};
            for (int li = 0; li < 15; ++li) {
                const int b = li / 3, j = li % 3;
                float* dst = blk[b % 2];
                int rc;
                if (li == 0) {
                    const bool three = !g.paf && !g.first;
                    rc = conv(ci[0], three ? net->f_cat3.p : net->f_cat.p, three ? kCat3 : kCat2, 0, dst, cs, 0, h, w, nullptr);
                } else if (j == 0) {
                    rc = conv(ci[li], blk[(b + 1) % 2], cs, 0, dst, cs, 0, h, w, nullptr);
                } else {
                    rc = conv(ci[li], dst, cs, (j - 1) * g.inner, dst, cs, j * g.inner, h, w, nullptr);
                }
                if (rc) return 1;
            }
            if (conv(ci[15], net->f_x.p, cs, 0, net->f_z.p, g.innerout, 0, h, w, nullptr)) return 1;
            if (conv(ci[16], net->f_z.p, g.innerout, 0, net->f_y.p, g.out, 0, h, w, net->out_f32[t].p)) return 1;
            // the next stages' inputs: an L2 head's PAF into cat[features, paf] (and the last one into
            // cat[features, heat, paf]), an L1 head's heat map into cat[features, heat, paf]
            if (g.paf) {
                CU(nchw_to_nhwc_f32_launch(net->out_f32[t].p, net->f_cat.p, n, kPaf, h, w, kCat2, kFeat, st));
                ++g_launches;
            }
            if (t == arch.l2 - 1 || !g.paf) {
                CU(nchw_to_nhwc_f32_launch(net->out_f32[t].p, net->f_cat3.p, n, g.out, h, w, kCat3,
                                           g.paf ? kFeat + kHeat : kFeat, st));
                ++g_launches;
            }
        }
        return 0;
    }
    for (int s = 1; s <= stages; ++s)
        for (int b = 0; b < 2; ++b) {
            const std::vector<int> ci = stage_convs(arch, s, b);
            const int nl = (int)ci.size();
            const float* in = net->f_cat.p;
            int in_cs = kCat, in_off = (s == 1) ? kPaf + kHeat : 0;
            float* bufs[2] = {net->f_x.p, net->f_y.p};
            for (int li = 0; li < nl; ++li) {
                const ConvSpec sp = arch.convs[ci[li]].s;
                const bool lastl = (li == nl - 1);
                float* nchw = lastl ? net->out_f32[2 * (s - 1) + b].p : nullptr;
                // last layer output goes to a scratch slice; the concat for the next stage is written after both
                // branches are done (the other branch still reads f_cat)
                float* dst = bufs[li & 1];
                if (conv(ci[li], in, in_cs, in_off, dst, sp.cout, 0, h, w, nchw)) return 1;
                in = dst; in_cs = sp.cout; in_off = 0;
            }
            if (b == 1 && s < stages) {
                CU(nchw_to_nhwc_f32_launch(net->out_f32[2 * (s - 1)].p, net->f_cat.p, n, kPaf, h, w, kCat, 0, st));
                CU(nchw_to_nhwc_f32_launch(net->out_f32[2 * (s - 1) + 1].p, net->f_cat.p, n, kHeat, h, w, kCat, kPaf, st));
                g_launches += 2;
            }
        }
    return 0;
}

}  // namespace

extern "C" {

const char* b200pose_last_error(void) { return g_err.c_str(); }
int b200pose_version(void) { return 100; }
long b200pose_launch_count(void) { return g_launches.load(); }

int b200pose_net_tensor_shape(int index, long dims[4]) {
    static const NetArch rtpose = rtpose_arch();
    return arch_tensor_shape(rtpose, index, dims);
}

int b200pose_openpose_num_tensors(int l2_stages, int l1_stages) {
    return op_valid(l2_stages, l1_stages) ? arch_num_tensors(openpose_arch(l2_stages, l1_stages)) : -1;
}

int b200pose_openpose_tensor_shape(int l2_stages, int l1_stages, int index, long dims[4]) {
    return op_valid(l2_stages, l1_stages) ? arch_tensor_shape(openpose_arch(l2_stages, l1_stages), index, dims) : -1;
}

static int net_create(b200pose_net** out, int cuda_device, NetArch arch) {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
        return cuda_fail("b200pose: no CUDA device available (this library has no CPU fallback)");
    CU(cudaSetDevice(cuda_device));
    cudaDeviceProp prop;
    CU(cudaGetDeviceProperties(&prop, cuda_device));
    if (prop.major != 9 || prop.minor != 0)
        return fail("b200pose: built for sm_90a (H100); device is sm_%d%d", prop.major, prop.minor);
    b200pose_net* net = new b200pose_net();
    net->device = cuda_device;
    net->num_sms = prop.multiProcessorCount;
    net->arch = std::move(arch);
    net->stages = net->arch.stages;
    const int nc = (int)net->arch.convs.size();
    net->host_w.resize(nc);
    net->host_b.resize(nc);
    net->host_slope.resize(nc);
    net->d_w.resize(nc);
    net->d_b.resize(nc);
    net->d_slope.resize(nc);
    net->have.assign(arch_num_tensors(net->arch), false);
    const char* gr = getenv("B200POSE_GRAPH");
    net->use_graph = !(gr && gr[0] == '0');
    *out = net;
    return 0;
}

int b200pose_net_create(b200pose_net** out, int cuda_device) { return net_create(out, cuda_device, rtpose_arch()); }

int b200pose_net_create_openpose(b200pose_net** out, int cuda_device, int l2_stages, int l1_stages) {
    if (!op_valid(l2_stages, l1_stages))
        return fail("OpenPose_Model(%d, %d): stages must be l2 >= 1, l1 >= 1, l2 + l1 <= %d", l2_stages, l1_stages,
                    kOpMaxStages);
    return net_create(out, cuda_device, openpose_arch(l2_stages, l1_stages));
}

void b200pose_net_destroy(b200pose_net* net) {
    if (!net) return;
    cudaSetDevice(net->device);
    delete net;
}

int b200pose_net_set_tensor(b200pose_net* net, int index, const float* host_data, long count) {
    if (!net || !host_data) return fail("set_tensor: null pointer");
    long dims[4];
    const int nd = arch_tensor_shape(net->arch, index, dims);
    const std::string who = is_openpose(net) ? net->arch.name + ": " : "";
    if (nd < 0) return fail("%stensor index %d out of range", who.c_str(), index);
    long expect = 1;
    for (int i = 0; i < nd; ++i) expect *= dims[i];
    if (count != expect) return fail("%stensor %d: got %ld elements, expected %ld", who.c_str(), index, count, expect);
    int ci, kind;
    arch_tensor(net->arch, index, &ci, &kind);
    std::vector<float>& dst = kind == 0 ? net->host_w[ci] : (kind == 1 ? net->host_b[ci] : net->host_slope[ci]);
    dst.assign(host_data, host_data + count);
    net->have[index] = true;
    net->finalized = false;
    return 0;
}

int b200pose_net_finalize(b200pose_net* net) {
    if (!net) return fail("null net");
    CU(cudaSetDevice(net->device));
    for (int i = 0; i < (int)net->have.size(); ++i)
        if (!net->have[i]) return fail("state_dict tensor %d was never set", i);
    for (size_t i = 0; i < net->arch.convs.size(); ++i) {
        // freed first, not reused: cudaFree synchronises the device, so a forward in flight on another stream has
        // stopped reading the weights before the synchronous copies below overwrite them
        net->d_w[i].release();
        net->d_b[i].release();
        net->d_slope[i].release();
        CU(net->d_w[i].ensure(net->host_w[i].size()));
        CU(net->d_b[i].ensure(net->host_b[i].size()));
        CU(net->d_slope[i].ensure(net->host_slope[i].size()));
        CU(cudaMemcpy(net->d_w[i].p, net->host_w[i].data(), net->host_w[i].size() * 4, cudaMemcpyHostToDevice));
        CU(cudaMemcpy(net->d_b[i].p, net->host_b[i].data(), net->host_b[i].size() * 4, cudaMemcpyHostToDevice));
        if (!net->host_slope[i].empty())
            CU(cudaMemcpy(net->d_slope[i].p, net->host_slope[i].data(), net->host_slope[i].size() * 4, cudaMemcpyHostToDevice));
    }
    net->tc.clear();
    for (const ArchLayer& l : net->arch.layers) net->tc.push_back(make_tc_layer(net->arch, l));
    for (TcLayer& L : net->tc)
        if (ensure_packed(net, L, TcFormat::kBf16)) return 1;
    net->last = LastForward();
    drop_graphs(net);
    net->plan = nullptr;
    net->plans.clear();      // the plans point at the previous packed weights
    net->finalized = true;
    return 0;
}

// Entries of outputs[12] for stages the net does not run must be NULL: a caller must not read a map no stage wrote as if
// it were fresh.
static int check_outputs(const b200pose_net* net, float* const* outputs) {
    for (int i = net->arch.out[net->stages].maps; outputs && i < 12; ++i)
        if (outputs[i]) {
            if (is_openpose(net))
                return fail("outputs[%d] must be NULL: %s writes %d maps", i, net->arch.name.c_str(), net->arch.out[net->stages].maps);
            return fail("outputs[%d] must be NULL: the net runs %d stage(s), stage %d does not run", i, net->stages, i / 2 + 1);
        }
    return 0;
}

// OpenPose_Model nets run the bf16, bf16x3 and fp32 modes; the fp8 and fp16 modes (their per-launch tables follow
// rtpose's launch list) are refused before anything is enqueued.
static int check_mode(const b200pose_net* net, int mode) {
    if (is_openpose(net) && (mode == B200POSE_MODE_FP8 || mode == B200POSE_MODE_FP16))
        return fail("%s runs modes bf16, bf16x3 and fp32, not %s", net->arch.name.c_str(),
                    mode == B200POSE_MODE_FP8 ? "fp8" : "fp16");
    return 0;
}

// ext: device extents table of a ragged batch (DESIGN.md §1), or null
static int net_forward_impl(b200pose_net* net, const void* input, int in_u8, int input_on_device, int n, int H, int W,
                            int mode, float* const* outputs, int outputs_on_device, cudaStream_t st, bool sync_host,
                            const int* ext = nullptr) {
    if (!net || !net->finalized) return fail("net not finalized");
    if (n < 1 || H < 8 || W < 8 || (H % 8) || (W % 8)) return fail("input must be [n,3,H,W] with H, W multiples of 8");
    if (int rc = check_outputs(net, outputs)) return rc;
    if (int rc = check_mode(net, mode)) return rc;
    const int stages = net->stages;
    CU(cudaSetDevice(net->device));
    const void* d_in = input;
    const size_t elems = (size_t)n * 3 * H * W;
    if (!input_on_device) {
        if (in_u8) {
            CU(net->in_stage_u8.ensure(elems));
            CU(cudaMemcpyAsync(net->in_stage_u8.p, input, elems, cudaMemcpyHostToDevice, st));
            d_in = net->in_stage_u8.p;
        } else {
            CU(net->in_stage.ensure(elems));
            CU(cudaMemcpyAsync(net->in_stage.p, input, elems * 4, cudaMemcpyHostToDevice, st));
            d_in = net->in_stage.p;
        }
    }
    int rc, first_u8 = 0;     // the uint8 normalisation conv1_1 fuses (tensor-core formats)
    TcFormat fmt = TcFormat::kBf16;
    if (mode == B200POSE_MODE_FP32) {
        if (in_u8) {   // parity mode: materialise rtpose_preprocess, then the fp32 path
            CU(net->f_u8.ensure(elems));
            CU(u8hwc_to_f32nchw_launch(static_cast<const unsigned char*>(d_in), net->f_u8.p, n, H, W, net->preprocess, ext, st));
            ++g_launches;
            rc = forward_fp32(net, net->f_u8.p, n, H, W, stages, st, ext);
        } else rc = forward_fp32(net, static_cast<const float*>(d_in), n, H, W, stages, st, ext);
    } else {
        if (mode == B200POSE_MODE_BF16X3) fmt = TcFormat::kBf16x3;
        else if (mode == B200POSE_MODE_FP8) fmt = TcFormat::kFp8;
        else if (mode == B200POSE_MODE_FP16) fmt = TcFormat::kFp16;     // every other mode runs bf16
        first_u8 = in_u8 ? net->preprocess : 0;
        rc = forward_tc(net, d_in, first_u8, n, H, W, fmt, stages, st, ext);
    }
    if (rc) return rc;
    net->last = LastForward{n, H, W, mode == B200POSE_MODE_FP32, fmt, stages, d_in, first_u8, ext,
                            ext ? net->ext_host : std::vector<int>()};
    if (outputs) {
        const size_t px8 = (size_t)n * (H / 8) * (W / 8);
        for (int i = 0; i < net->arch.out[stages].maps; ++i)
            if (outputs[i])
                CU(cudaMemcpyAsync(outputs[i], net->out_f32[i].p, px8 * net->arch.map_ch[i] * 4,
                                   outputs_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, st));
    }
    if (sync_host && (!input_on_device || (outputs && !outputs_on_device))) CU(cudaStreamSynchronize(st));
    return 0;
}

int b200pose_net_forward(b200pose_net* net, const float* input, int input_on_device, int n, int H, int W, int mode,
                         float* const* outputs, int outputs_on_device, void* cuda_stream) {
    return net_forward_impl(net, input, 0, input_on_device, n, H, W, mode, outputs, outputs_on_device,
                            reinterpret_cast<cudaStream_t>(cuda_stream), true);
}

int b200pose_net_forward_u8(b200pose_net* net, const unsigned char* images, int input_on_device, int n, int H, int W,
                            int mode, float* const* outputs, int outputs_on_device, void* cuda_stream) {
    return net_forward_impl(net, images, 1, input_on_device, n, H, W, mode, outputs, outputs_on_device,
                            reinterpret_cast<cudaStream_t>(cuda_stream), true);
}

// ------------------------------------------------------------------------------------------------ ragged batches
// Validates the padded sizes of a ragged batch (DESIGN.md §1) and returns its canvas.
static int ragged_canvas(int n, const int* hw, int* Hc, int* Wc) {
    if (n < 1 || n > kMaxRagged) return fail("ragged batch: %d images (1 .. %d)", n, kMaxRagged);
    if (!hw) return fail("ragged batch: null size table");
    *Hc = *Wc = 0;
    for (int i = 0; i < n; ++i) {
        const int H = hw[2 * i], W = hw[2 * i + 1];
        if (H < 8 || W < 8 || (H % 8) || (W % 8)) return fail("ragged batch: image %d is %d x %d (multiples of 8 needed)", i, H, W);
        if (H > *Hc) *Hc = H;
        if (W > *Wc) *Wc = W;
    }
    return 0;
}

// Writes the extents of the next ragged forward into the net's fixed table (stream-ordered after the previous forward).
static int upload_ext(b200pose_net* net, const std::vector<int>& ext, cudaStream_t st) {
    CU(net->d_ext.ensure((size_t)kMaxRagged * 2));
    CU(cudaMemcpyAsync(net->d_ext.p, ext.data(), ext.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    net->ext_host = ext;
    return 0;
}

static int upload_frames(b200pose_net* net, const std::vector<RaggedFrame>& frames, cudaStream_t st) {
    CU(net->d_frames.ensure(frames.size()));
    CU(cudaMemcpyAsync(net->d_frames.p, frames.data(), frames.size() * sizeof(RaggedFrame), cudaMemcpyHostToDevice, st));
    return 0;
}

// fp16 overflow rows a fused run keeps: one per forward, at most 16 scales
constexpr int kMaxOvfRows = 16;

// A batch of raw uint8 frames packed back to back, cropped for one destination size: frame table (flip: the mirrored
// frames follow the originals, in the staging buffer and in both tables), padded extents and canvas, the frames' total
// and largest size in bytes.  A uniform batch (frames of one size) keeps `ext` empty: its forward and post-processing get
// no extents table.
struct RawBatch {
    std::vector<RaggedFrame> tab;
    std::vector<int> ext;
    int Hc = 0, Wc = 0;
    long long raw = 0, max_bytes = 0;
    bool ragged() const { return !ext.empty(); }
};

// Crops the nimg frames of c (sources at d_raw; frame table already in net->d_frames) into net->in_stage_u8 and runs
// the forward pass on them.
static int crop_and_forward(b200pose_net* net, const unsigned char* d_raw, int nimg, const RawBatch& c, int mode,
                            cudaStream_t st, float* const* outputs = nullptr, int outputs_on_device = 1,
                            bool sync_host = false) {
    CU(net->in_stage_u8.ensure((size_t)nimg * c.Hc * c.Wc * 3));
    if (launched(crop_frames_launch(d_raw, net->d_frames.p, nimg, net->in_stage_u8.p, c.Hc, c.Wc, st), "crop_frames_launch"))
        return 1;
    if (c.ragged() && upload_ext(net, c.ext, st)) return 1;
    return net_forward_impl(net, net->in_stage_u8.p, 1, 1, nimg, c.Hc, c.Wc, mode, outputs, outputs_on_device, st,
                            sync_host, c.ragged() ? net->d_ext.p : nullptr);
}

// Raw uint8 frames of `bytes` on the device: a device input in place, else a copy in net->raw_stage.  flip: always
// copied, with room for the mirror images behind the frames.
static int stage_raw(b200pose_net* net, const unsigned char* images, int on_device, size_t bytes, int flip,
                     cudaStream_t st, const unsigned char** d_raw) {
    *d_raw = images;
    if (on_device && !flip) return 0;
    CU(net->raw_stage.ensure(bytes * (flip ? 2 : 1)));
    CU(cudaMemcpyAsync(net->raw_stage.p, images, bytes, on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, st));
    *d_raw = net->raw_stage.p;
    return 0;
}

int b200pose_net_forward_ragged_u8(b200pose_net* net, const unsigned char* frames, int on_device, int n, const int* hw,
                                   int mode, float* const* outputs, int outputs_on_device, void* cuda_stream) {
    if (!net || !net->finalized) return fail("net not finalized");
    if (!frames) return fail("forward_ragged: null pointer");
    if (int rc = check_outputs(net, outputs)) return rc;
    if (int rc = check_mode(net, mode)) return rc;
    int Hc, Wc;
    if (int rc = ragged_canvas(n, hw, &Hc, &Wc)) return rc;
    CU(cudaSetDevice(net->device));
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    RawBatch c;
    c.tab.assign(n, RaggedFrame{});
    c.ext.assign(hw, hw + 2 * n);
    c.Hc = Hc;
    c.Wc = Wc;
    for (int i = 0; i < n; ++i) {
        c.tab[i].off = c.raw;
        c.tab[i].src_h = hw[2 * i];
        c.tab[i].src_w = hw[2 * i + 1];      // g.pad_h == 0: copied as it is
        c.raw += (long long)hw[2 * i] * hw[2 * i + 1] * 3;
    }
    const unsigned char* d_src;
    if (int rc = stage_raw(net, frames, on_device, (size_t)c.raw, 0, st, &d_src)) return rc;
    if (int rc = upload_frames(net, c.tab, st)) return rc;
    if (int rc = crop_and_forward(net, d_src, n, c, mode, st, outputs, outputs_on_device, true)) return rc;
    if (!on_device) CU(cudaStreamSynchronize(st));
    return 0;
}

int b200pose_net_set_preprocess(b200pose_net* net, int preprocess) {
    if (!net) return fail("null net");
    if (preprocess < 1 || preprocess > 4) return fail("preprocess must be 1 (rtpose), 2 (vgg), 3 (inception) or 4 (ssd)");
    net->preprocess = preprocess;
    return 0;
}

int b200pose_net_set_jpeg_progressive(b200pose_net* net, int on) {
    if (!net) return fail("null net");
    net->jpeg_progressive = on != 0;
    return 0;
}

int b200pose_net_get_jpeg_progressive(b200pose_net* net) {
    if (!net) return fail("null net"), -1;
    return net->jpeg_progressive ? 1 : 0;
}

int b200pose_net_set_stages(b200pose_net* net, int stages) {
    if (!net) return fail("null net");
    if (is_openpose(net))
        return fail("%s: the stage count is the architecture's (set at b200pose_net_create_openpose)", net->arch.name.c_str());
    if (stages < 1 || stages > kStages) return fail("stages must be 1 .. %d, got %d", kStages, stages);
    net->stages = stages;
    return 0;
}

// The last forward ran net->plan: a tensor-core forward has run since the last finalize.
static bool last_ran_plan(const b200pose_net* net) {
    const LastForward& l = net->last;
    const Plan* p = net->plan;
    return p && !l.fp32 && p->n == l.n && p->H == l.H && p->W == l.W && p->fmt == l.fmt && p->stages == l.stages;
}

int b200pose_net_profile(b200pose_net* net, float* ms, double* flops, int cap, void* cuda_stream) {
    if (!net || !last_ran_plan(net)) return -1;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    const Plan& p = *net->plan;
    const int n = p.n, H = p.H, W = p.W;
    const int total = (int)p.launches.size() + 1;
    if (cap < total) return -1;
    std::vector<Event> ev(total + 1);
    DevBuf<float> tmp;
    auto run = [&]() -> int {
        CU(cudaSetDevice(net->device));
        for (Event& e : ev) CU(cudaEventCreate(&e.h));
        const void* d_in = net->last.in;
        int in_u8 = net->last.in_u8;
        if (!d_in) {
            CU(tmp.ensure((size_t)n * 3 * H * W));
            CU(cudaMemsetAsync(tmp.p, 0, (size_t)n * 3 * H * W * 4, st));
            d_in = tmp.p;
            in_u8 = 0;
        }
        CU(cudaEventRecord(ev[0], st));
        const int rc = launch_forward_tc(net, d_in, in_u8, nullptr, total, st, false, ev.data() + 1);
        g_launches += total;
        if (rc) return rc;
        CU(cudaStreamSynchronize(st));
        for (int i = 0; i < total; ++i) CU(cudaEventElapsedTime(&ms[i], ev[i], ev[i + 1]));
        flops[0] = 2.0 * n * H * W * 27.0 * 64.0;
        for (size_t i = 0; i < p.launches.size(); ++i) flops[i + 1] = p.launches[i].flops;
        return 0;
    };
    return run() ? -1 : total;
}

int b200pose_net_debug_run(b200pose_net* net, int launches, void* cuda_stream) {
    if (!net || !last_ran_plan(net) || !net->last.in) return fail("debug_run: no tensor-core forward has run");
    if (launches < 0 || launches > 1 + (int)net->plan->launches.size())
        return fail("debug_run: %d launches out of range", launches);
    CU(cudaSetDevice(net->device));
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (launch_forward_tc(net, net->last.in, net->last.in_u8, net->last.ext, launches, st)) return 1;
    g_launches += launches;
    CU(cudaStreamSynchronize(st));
    return 0;
}

int b200pose_net_debug_launch(b200pose_net* net, int i, int* fields, int cap) {
    if (!net || !last_ran_plan(net)) return fail("debug_launch: no tensor-core forward has run");
    const Plan& p = *net->plan;
    // fields 0 .. 26 are required; the format field is written when there is room for it
    constexpr int kAll = B200POSE_DEBUG_LAUNCH_FORMAT + 1;
    const int nf = cap < kAll ? cap : kAll;
    if (i < 0 || i > (int)p.launches.size() || nf < B200POSE_DEBUG_LAUNCH_FIELDS || !fields)
        return fail("debug_launch: launch %d / capacity %d out of range", i, cap);
    int f[kAll] = {};
    if (i == 0) {     // conv1_1 (CUDA cores / mma.sync): the network input -> t1
        f[0] = -1; f[1] = 3; f[4] = T1; f[5] = kActC[T1]; f[8] = 64;
        f[10] = p.H; f[11] = p.W; f[12] = 3; f[14] = 1; f[15] = 64; f[16] = 1; f[17] = 1;
        f[19] = tc_planes(p.fmt) - 1; f[23] = f[24] = -1;
        f[26] = net->last.in_u8;
    } else {
        const PlanLaunch& l = p.launches[i - 1];
        const ConvTcArgs& a = l.a;
        f[0] = l.in; f[1] = net->arch.act_c[l.in]; f[2] = a.in_ch_base; f[3] = a.in_ch_group_stride;
        f[4] = l.out; f[5] = a.out_cstride; f[6] = a.out_ch_off[0]; f[7] = a.out_ch_off[1];
        f[8] = a.store_ch[0]; f[9] = a.store_ch[1];
        f[10] = a.H; f[11] = a.W; f[12] = a.ksize; f[13] = a.cin_blocks; f[14] = a.groups; f[15] = a.n_tile;
        f[16] = a.n_tiles; f[17] = a.relu; f[18] = a.pool; f[19] = a.split; f[20] = tc_chunked(a.fmt) ? 1 : 0; f[21] = a.pdl; f[22] = a.tps;
        f[23] = l.f32[0]; f[24] = l.f32[1];
    }
    f[25] = p.n;
    f[B200POSE_DEBUG_LAUNCH_FORMAT] = tc_binary16(p.fmt) ? 1 : 0;
    for (int k = 0; k < nf; ++k) fields[k] = f[k];
    return nf;
}

int b200pose_net_debug_read(b200pose_net* net, int buf, int lo_plane, int img0, int count, void* host, long bytes) {
    if (!net || !last_ran_plan(net)) return fail("debug_read: no tensor-core forward has run");
    const int n = net->plan->n, H = net->plan->H, W = net->plan->W;
    if (img0 < 0 || count < 1 || img0 + count > n || !host) return fail("debug_read: images [%d, %d) out of range", img0, img0 + count);
    const char* src = nullptr;
    size_t per = 0;
    if (buf >= 0 && buf < kNumAct) {
        if (lo_plane && tc_planes(net->plan->fmt) < 2) return fail("debug_read: residual planes exist in bf16x3 mode only");
        per = (size_t)(H / kActDiv[buf]) * (W / kActDiv[buf]) * net->arch.act_c[buf] * 2;
        src = reinterpret_cast<const char*>((lo_plane ? net->act_lo : net->act)[buf].p);
    } else if (buf >= kNumAct && buf < kNumAct + 12 && !lo_plane) {
        const int m = buf - kNumAct;
        if (m >= net->arch.out[net->last.stages].maps)
            return fail("debug_read: stage map %d was not written by the last forward (%d stages)", m, net->last.stages);
        per =(size_t)(H / 8) * (W / 8) * net->arch.map_ch[m] * 4;
        src = reinterpret_cast<const char*>(net->out_f32[m].p);
    } else {
        return fail("debug_read: no buffer %d (plane %d)", buf, lo_plane);
    }
    if (bytes < (long)(per * count)) return fail("debug_read: %ld bytes given, %zu needed", bytes, per * count);
    CU(cudaSetDevice(net->device));
    CU(cudaMemcpy(host, src + per * img0, per * count, cudaMemcpyDeviceToHost));
    return 0;
}

int b200pose_net_debug_fp8(b200pose_net* net, int launch, int* act_exp, int n_img, int* w_exp, int cap) {
    if (!net || !last_ran_plan(net) || net->plan->fmt != TcFormat::kFp8) { fail("debug_fp8: no fp8 forward has run"); return -1; }
    const Plan& p = *net->plan;
    if (launch < 1 || launch > (int)p.launches.size() || n_img != p.n || !act_exp || !w_exp) {
        fail("debug_fp8: launch %d / images %d out of range", launch, n_img);
        return -1;
    }
    const ConvTcArgs& a = p.launches[launch - 1].a;
    const int rows = a.groups * a.n_tiles * a.n_tile;
    if (cap < rows) { fail("debug_fp8: %d rows, capacity %d", rows, cap); return -1; }
    cudaError_t e = cudaSetDevice(net->device);
    if (e == cudaSuccess) e = cudaMemcpy(act_exp, a.ea_out, p.n * sizeof(int), cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) { cuda_fail("debug_fp8: reading the exponent table: %s", cudaGetErrorString(e)); return -1; }
    const TcLayer& L = net->tc[launch - 1];
    for (int r = 0; r < rows; ++r) w_exp[r] = L.h_w_exp[r];
    return rows;
}

int b200pose_net_overflow(b200pose_net* net, int* flags, int n, void* cuda_stream) {
    if (!net || !flags) { fail("overflow: null pointer"); return -1; }
    if (net->last.n == 0) { fail("overflow: no forward has run"); return -1; }
    if (n != net->last.n) { fail("overflow: %d images asked, the last forward ran %d", n, net->last.n); return -1; }
    std::vector<unsigned> h(n, 0u);
    cudaError_t e = cudaSetDevice(net->device);
    if (e == cudaSuccess) e = cudaStreamSynchronize(reinterpret_cast<cudaStream_t>(cuda_stream));
    if (e == cudaSuccess && !net->last.fp32 && tc_aux(net->last.fmt) == TcAux::kOverflow)
        e = cudaMemcpy(h.data(), net->ovf.p, n * sizeof(unsigned), cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) { cuda_fail("overflow: %s", cudaGetErrorString(e)); return -1; }
    int flagged = 0;
    for (int i = 0; i < n; ++i) flagged += (flags[i] = h[i] != 0);
    return flagged;
}

int b200pose_net_last_maps(b200pose_net* net, const float** paf, const float** heat, int* n, int* h, int* w) {
    if (!net || net->last.n == 0) return fail("no forward has run");
    *paf = last_paf(net); *heat = last_heat(net);
    *n = net->last.n; *h = net->last.H / 8; *w = net->last.W / 8;
    return 0;
}

// ------------------------------------------------------------------------------------------------ post
int b200pose_post_create(b200pose_post** out, int cuda_device, int batch_cap, int peak_cap, int human_cap) {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
        return cuda_fail("b200pose: no CUDA device available (this library has no CPU fallback)");
    CU(cudaSetDevice(cuda_device));
    std::unique_ptr<b200pose_post> p(new b200pose_post());
    p->device = cuda_device;
    // candidate-key pool (DESIGN §1): min(batch_cap x 16 Mi, 1 Gi) 8-byte entries, i.e. 128 MB per image of the batch and
    // at most 8 GiB; exhausting it sets a status bit (a loud error in the Python layer)
    const long pool = (long)batch_cap * (16L << 20) < (1L << 30) ? (long)batch_cap * (16L << 20) : (1L << 30);
    cudaError_t e = post_alloc(p->pb, batch_cap, peak_cap, human_cap, pool);
    if (e != cudaSuccess) return cuda_fail("post_alloc failed: %s", cudaGetErrorString(e));
    CU(cudaStreamCreateWithFlags(&p->s2.h, cudaStreamNonBlocking));
    for (Event* ev : {&p->ev_limbs, &p->ev_asm, &p->ev_maps, &p->ev_fetch[0], &p->ev_fetch[1], &p->ev_ld[0], &p->ev_ld[1],
                      &p->ev_draw})
        CU(cudaEventCreateWithFlags(&ev->h, cudaEventDisableTiming));
    for (int b = 0; b < 2; ++b) {
        CU(p->hp_nh[b].alloc(batch_cap, cudaHostAllocDefault));
        CU(p->hp_status[b].alloc(batch_cap, cudaHostAllocDefault));
        CU(p->hp_counts[b].alloc((size_t)batch_cap * 18, cudaHostAllocDefault));
        // written by assemble_kernel (same pointer on the device: unified addressing)
        CU(p->hp_humans[b].alloc((size_t)batch_cap * human_cap * kHumanFloats, cudaHostAllocMapped | cudaHostAllocPortable));
        CU(p->d_ext[b].ensure((size_t)batch_cap * 2));
        CU(p->hp_ovf[b].alloc((size_t)kMaxOvfRows * 2 * batch_cap, cudaHostAllocDefault));
        CU(p->hp_jpeg[b].alloc(batch_cap, cudaHostAllocDefault));
        CU(p->hp_png[b].alloc(batch_cap, cudaHostAllocDefault));
    }
    *out = p.release();
    return 0;
}

void b200pose_post_destroy(b200pose_post* p) {
    if (!p) return;
    cudaSetDevice(p->device);
    delete p;
}

// The settings a run launches with: null (the kernels compiled with the reference's constants) when they are the
// defaults, so default runs execute exactly the kernels they always did.
static const PostParams* run_params(const b200pose_post* p) {
    const PostParams& q = p->params;
    const bool dflt = q.paf_thresh == DefaultPostParams::paf_thresh && q.paf_samples == DefaultPostParams::paf_samples &&
                      q.paf_min_above == DefaultPostParams::paf_min_above && q.min_parts == DefaultPostParams::min_parts &&
                      q.min_person_score == DefaultPostParams::min_person_score;
    return dflt ? nullptr : &q;
}

// After the limbs kernel was enqueued on `st`: assembly + result copies on the second stream.  prm: as for post_limbs.
static int enqueue_assemble_and_fetch(b200pose_post* p, int n, cudaStream_t st, const PostParams* prm) {
    CU(cudaEventRecord(p->ev_limbs, st));
    CU(cudaStreamWaitEvent(p->s2, p->ev_limbs, 0));
    const int b = (int)(p->runs & 1);
    // the assembly kernel writes the person rows straight into this run's pinned host slot (unified addressing): only the
    // rows that exist cross PCIe, instead of a copy of the full-capacity buffer (4.8 MB per step at batch 32)
    p->pb.humans_out = p->hp_humans[b].p;
    if (launched(post_assemble(p->pb, n, p->s2, prm), "post_assemble")) return 1;
    CU(cudaEventRecord(p->ev_asm, p->s2));
    const PostBuffers& pb = p->pb;
    CU(cudaMemcpyAsync(p->hp_nh[b].p, pb.n_humans, n * sizeof(int), cudaMemcpyDeviceToHost, p->s2));
    CU(cudaMemcpyAsync(p->hp_status[b].p, pb.status, n * sizeof(int), cudaMemcpyDeviceToHost, p->s2));
    CU(cudaMemcpyAsync(p->hp_counts[b].p, pb.counts, (size_t)n * 18 * sizeof(int), cudaMemcpyDeviceToHost, p->s2));
    CU(cudaEventRecord(p->ev_fetch[b], p->s2));
    p->slot_n[b] = n;
    p->ovf_rows[b] = p->ovf_pending;
    p->ovf_imgs[b] = p->ovf_pending_imgs;
    p->ovf_pending = 0;
    p->jpeg_imgs[b] = p->jpeg_pending;
    p->jpeg_pending = 0;
    p->png_imgs[b] = p->png_pending;
    p->png_pending = 0;
    p->runs += 1;
    p->h_px.clear();
    return 0;
}

static int check_batch(const b200pose_post* p, int n) {
    if (n > p->pb.batch_cap) return fail("batch %d exceeds post batch_cap %d", n, p->pb.batch_cap);
    return 0;
}

// ext: device extents table of a ragged batch (h x w is then its canvas at the maps' resolution), or null
// up: the factor from the maps to the peak coordinates (8 for every fused run)
static int post_run_dev(b200pose_post* p, const float* d_heat, const float* d_paf, int layout, int n, int h, int w,
                        float thresh, cudaStream_t st, const int* ext = nullptr, int up = 8) {
    if (int rc = check_batch(p, n)) return rc;
    if (up < 1 || up > kMaxUpsample) return fail("post_run: upsample must be 1 .. %d, got %d", kMaxUpsample, up);
    if ((long)h * up > kMaxUpCoord || (long)w * up > kMaxUpCoord)
        return fail("post_run: maps of %d x %d at upsample %d give %ld x %ld pixels, above %d", h, w, up, (long)h * up,
                    (long)w * up, kMaxUpCoord);
    const int slot = (int)(p->runs & 1);
    if (p->have_ld[slot]) CU(cudaStreamWaitEvent(st, p->ev_ld[slot], 0));   // run i-2 is done with this slot
    if (ext) {
        CU(cudaMemcpyAsync(p->d_ext[slot].p, ext, (size_t)n * 2 * sizeof(int), cudaMemcpyDeviceToDevice, st));
        ext = p->d_ext[slot].p;
    }
    // private copy of the maps (15 MB at batch 32) so that the next forward may overwrite the network's output
    // buffers while this run's post-processing is still reading; everything after the copy runs on s2
    const size_t eh = (size_t)n * 19 * h * w, ep = (size_t)n * 38 * h * w;
    CU(p->ov_maps[slot].ensure(eh + ep));
    CU(cudaMemcpyAsync(p->ov_maps[slot].p, d_heat, eh * 4, cudaMemcpyDeviceToDevice, st));
    CU(cudaMemcpyAsync(p->ov_maps[slot].p + eh, d_paf, ep * 4, cudaMemcpyDeviceToDevice, st));
    CU(cudaEventRecord(p->ev_maps, st));
    CU(cudaStreamWaitEvent(p->s2, p->ev_maps, 0));
    d_heat = p->ov_maps[slot].p;
    d_paf = p->ov_maps[slot].p + eh;
    cudaStream_t ps = p->s2;       // the stream peaks / limbs run on
    // the previous run's assembly (second stream) still reads the peak / connection buffers this run overwrites, and
    // its D2H copies of status / counts (enqueued after the assembly) must not race with this run's memset + peaks:
    // wait for the event recorded after those copies
    if (p->runs > 0) CU(cudaStreamWaitEvent(ps, p->ev_fetch[(p->runs - 1) & 1], 0));
    cudaError_t e;
    const PostParams* prm = run_params(p);
    if (layout == 0) {
        e = post_peaks(p->pb, n, d_heat, (long)19 * h * w, (long)h * w, w, 1, h, w, thresh, ps, ext, up, p->refine);
        if (launched(e, "post_peaks")) return 1;
        e = post_limbs(p->pb, n, d_paf, (long)38 * h * w, (long)h * w, w, 1, 3, h * up, w, h, ps, ext, prm,
                       p->score_blocks, p->sort_blocks, up);
    } else {
        if (ext) return fail("post_run: ragged batches need the planar (layout 0) maps");
        e = post_peaks(p->pb, n, d_heat, (long)19 * h * w, 1, (long)w * 19, 19, h, w, thresh, ps, nullptr, up, p->refine);
        if (launched(e, "post_peaks")) return 1;
        e = post_limbs(p->pb, n, d_paf, (long)38 * h * w, 1, (long)w * 38, 38, 3, h * up, w, h, ps, nullptr, prm,
                       p->score_blocks, p->sort_blocks, up);
    }
    if (launched(e, "post_limbs")) return 1;
    CU(cudaEventRecord(p->ev_ld[slot], ps));
    p->have_ld[slot] = true;
    p->hw_h = h; p->hw_w = w;
    return enqueue_assemble_and_fetch(p, n, ps, prm);
}

int b200pose_post_run(b200pose_post* p, const float* heat, const float* paf, int on_device, int layout, int n, int h,
                      int w, float thresh, void* cuda_stream) {
    return b200pose_post_run_scaled(p, heat, paf, on_device, layout, n, h, w, 8, thresh, cuda_stream);
}

int b200pose_post_run_scaled(b200pose_post* p, const float* heat, const float* paf, int on_device, int layout, int n,
                             int h, int w, int upsample, float thresh, void* cuda_stream) {
    if (!p) return fail("null post");
    if (upsample < 1 || upsample > kMaxUpsample)
        return fail("post_run: upsample must be 1 .. %d, got %d", kMaxUpsample, upsample);
    if ((long)h * upsample > kMaxUpCoord || (long)w * upsample > kMaxUpCoord)
        return fail("post_run: maps of %d x %d at upsample %d give %ld x %ld pixels, above %d", h, w, upsample,
                    (long)h * upsample, (long)w * upsample, kMaxUpCoord);
    CU(cudaSetDevice(p->device));
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    p->ovf_pending = 0;      // maps from the caller: no network ran in this run
    p->jpeg_pending = 0;
    p->png_pending = 0;
    const float *dh = heat, *dp = paf;
    if (!on_device) {
        CU(p->d_heat.ensure((size_t)n * 19 * h * w));
        CU(p->d_paf.ensure((size_t)n * 38 * h * w));
        CU(cudaMemcpyAsync(p->d_heat.p, heat, (size_t)n * 19 * h * w * 4, cudaMemcpyHostToDevice, st));
        CU(cudaMemcpyAsync(p->d_paf.p, paf, (size_t)n * 38 * h * w * 4, cudaMemcpyHostToDevice, st));
        dh = p->d_heat.p; dp = p->d_paf.p;
    }
    return post_run_dev(p, dh, dp, layout, n, h, w, thresh, st, nullptr, upsample);
}

int b200pose_post_set_refine(b200pose_post* p, int mode) {
    if (!p) return fail("null post");
    if (mode < B200POSE_REFINE_NONE || mode > B200POSE_REFINE_CUBIC_GAUSS)
        return fail("post_set_refine: mode must be %d (none), %d (cubic) or %d (cubic+gauss), got %d", B200POSE_REFINE_NONE,
                    B200POSE_REFINE_CUBIC, B200POSE_REFINE_CUBIC_GAUSS, mode);
    p->refine = mode;
    return 0;
}

int b200pose_post_get_refine(b200pose_post* p) {
    if (!p) return fail("null post");
    return p->refine;
}

int b200pose_post_default_params(b200pose_post_params* out) {
    if (!out) return fail("post_default_params: null pointer");
    *out = b200pose_post_params{DefaultPostParams::paf_thresh, DefaultPostParams::paf_samples,
                                DefaultPostParams::paf_min_above, DefaultPostParams::min_parts,
                                DefaultPostParams::min_person_score};
    return 0;
}

int b200pose_post_set_params(b200pose_post* p, const b200pose_post_params* in) {
    if (!p) return fail("null post");
    b200pose_post_params q;
    if (in) q = *in;
    else b200pose_post_default_params(&q);
    const PostParams v{q.paf_thresh, q.paf_samples, q.paf_min_above, q.min_parts, q.min_person_score};
    char msg[160];
    if (!post_params_check(v, msg, sizeof(msg))) return fail("post params: %s", msg);
    p->params = v;
    return 0;
}

int b200pose_post_get_params(b200pose_post* p, b200pose_post_params* out) {
    if (!p || !out) return fail("post_get_params: null pointer");
    const PostParams& q = p->params;
    *out = b200pose_post_params{q.paf_thresh, q.paf_samples, q.paf_min_above, q.min_parts, q.min_person_score};
    return 0;
}

int b200pose_post_set_grids(b200pose_post* p, int score_blocks, int sort_blocks) {
    if (!p) return fail("null post");
    if (score_blocks < 0 || score_blocks > 65535)
        return fail("post_set_grids: score_blocks %d is outside 0 .. 65535", score_blocks);
    if (sort_blocks < 0 || sort_blocks > 65535)
        return fail("post_set_grids: sort_blocks %d is outside 0 .. 65535", sort_blocks);
    p->score_blocks = score_blocks;
    p->sort_blocks = sort_blocks;
    return 0;
}

long b200pose_post_last_ticket(b200pose_post* p) { return p ? p->runs - 1 : -1; }

int b200pose_post_select(b200pose_post* p, long ticket) {
    if (!p) return fail("null post");
    if (ticket < 0 || ticket >= p->runs || ticket < p->runs - 2) return fail("ticket %ld is not one of the last two runs", ticket);
    CU(cudaSetDevice(p->device));
    CU(cudaEventSynchronize(p->ev_fetch[ticket & 1]));
    p->cur = (int)(ticket & 1);
    p->cur_ticket = ticket;
    return 0;
}

int b200pose_post_sync(b200pose_post* p) {
    if (!p) return fail("null post");
    if (p->runs == 0) return fail("no run submitted");
    return b200pose_post_select(p, p->runs - 1);
}

int b200pose_post_status_accum(b200pose_post* p, int reset) {
    // OR of the status words of every image of every run since the last reset: lets a caller that keeps runs in flight
    // (and only reads some of them back) prove that NO run overflowed a capacity
    if (!p) return -1;
    std::vector<int> h(p->pb.batch_cap);
    cudaError_t e = cudaSetDevice(p->device);
    if (e == cudaSuccess) e = cudaStreamSynchronize(p->s2);
    if (e == cudaSuccess) e = cudaMemcpy(h.data(), p->pb.status_acc, h.size() * sizeof(int), cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && reset) e = cudaMemset(p->pb.status_acc, 0, h.size() * sizeof(int));
    if (e != cudaSuccess) { cuda_fail("status_accum: %s", cudaGetErrorString(e)); return -1; }
    int acc = 0;
    for (int v : h) acc |= v;
    return acc;
}

int b200pose_post_debug_sort(b200pose_post* p, const unsigned long long* keys, int n, unsigned long long* out) {
    if (!p || !keys || !out) return fail("debug_sort: null pointer");
    CU(cudaSetDevice(p->device));
    CU(cudaStreamSynchronize(p->s2));
    return launched(post_debug_sort(p->pb, keys, n, out, nullptr, p->sort_blocks), "post_debug_sort", 2);
}

int b200pose_post_debug_connections(b200pose_post* p, int img, int limb, int* a, int* b, float* s, int cap) {
    // valid for the LATEST run only (reads the device connection lists, which the next run overwrites); a count can be
    // 1, so errors return -1
    if (!p || !a || !b || !s) return -fail("debug_connections: null pointer");
    if (p->runs == 0) return -fail("debug_connections: no run submitted");
    if (b200pose_post_select(p, p->runs - 1)) return -1;
    if (img < 0 || img >= p->slot_n[p->cur] || limb < 0 || limb >= kNumLimb || cap < 0)
        return -fail("debug_connections: image %d of %d, limb %d, cap %d", img, p->slot_n[p->cur], limb, cap);
    const PostBuffers& pb = p->pb;
    const long li = (long)img * kNumLimb + limb;
    int cnt = 0;
    cudaError_t e = cudaMemcpy(&cnt, pb.conn_cnt + li, sizeof(int), cudaMemcpyDeviceToHost);
    const size_t k = (size_t)(cnt < cap ? cnt : cap);
    if (e == cudaSuccess && k > 0) e = cudaMemcpy(a, pb.conn_a + li * pb.peak_cap, k * sizeof(int), cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && k > 0) e = cudaMemcpy(b, pb.conn_b + li * pb.peak_cap, k * sizeof(int), cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && k > 0) e = cudaMemcpy(s, pb.conn_s + li * pb.peak_cap, k * sizeof(float), cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) return -cuda_fail("debug_connections: %s", cudaGetErrorString(e));
    return cnt;
}

int b200pose_post_debug(b200pose_post* p, unsigned long long* out, int n, int reset) {
    if (!p || n > 16) return -1;
    cudaError_t e = cudaMemcpy(out, p->pb.dbg, n * sizeof(unsigned long long), cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && reset) e = cudaMemset(p->pb.dbg, 0, 16 * sizeof(unsigned long long));
    if (e != cudaSuccess) { cuda_fail("post_debug: %s", cudaGetErrorString(e)); return -1; }
    return 0;
}

int b200pose_post_debug_maps(b200pose_post* p, float* heat, long heat_floats, float* paf, long paf_floats) {
    if (!p || !heat || !paf) return fail("debug_maps: null pointer");
    if (heat_floats < 0 || paf_floats < 0 || (size_t)heat_floats > p->d_heat.n || (size_t)paf_floats > p->d_paf.n)
        return fail("debug_maps: %ld / %ld floats asked, %zu / %zu held", heat_floats, paf_floats, p->d_heat.n, p->d_paf.n);
    CU(cudaSetDevice(p->device));
    CU(cudaDeviceSynchronize());
    CU(cudaMemcpy(heat, p->d_heat.p, (size_t)heat_floats * 4, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(paf, p->d_paf.p, (size_t)paf_floats * 4, cudaMemcpyDeviceToHost));
    return 0;
}
static int post_ready(b200pose_post* p, int img) {
    if (!p) return 0;
    if (p->cur_ticket < 0 && b200pose_post_sync(p)) return 0;
    return img >= 0 && img < p->slot_n[p->cur];
}
int b200pose_post_num_humans(b200pose_post* p, int img) { return post_ready(p, img) ? p->hp_nh[p->cur].p[img] : -1; }
int b200pose_post_status(b200pose_post* p, int img) { return post_ready(p, img) ? p->hp_status[p->cur].p[img] : -1; }
int b200pose_post_overflow(b200pose_post* p, int img) {
    if (!post_ready(p, img)) return -1;
    const int b = p->cur, n = p->slot_n[b];
    const unsigned* h = p->hp_ovf[b].p;
    for (int k = 0; k < p->ovf_rows[b]; ++k, h += 2 * (size_t)p->pb.batch_cap)
        if (h[img] || (p->ovf_imgs[b] == 2 * n && h[n + img])) return 1;
    return 0;
}
int b200pose_post_jpeg_status(b200pose_post* p, int img) {
    if (!post_ready(p, img)) return -1;
    return img < p->jpeg_imgs[p->cur] ? (int)p->hp_jpeg[p->cur].p[img] : 0;
}
int b200pose_post_png_status(b200pose_post* p, int img) {
    if (!post_ready(p, img)) return -1;
    return img < p->png_imgs[p->cur] ? (int)p->hp_png[p->cur].p[img] : 0;
}
int b200pose_post_get_humans(b200pose_post* p, int img, float* out, int max_humans) {
    if (!post_ready(p, img)) return -1;
    const int n = p->hp_nh[p->cur].p[img] < max_humans ? p->hp_nh[p->cur].p[img] : max_humans;
    memcpy(out, p->hp_humans[p->cur].p + (size_t)img * p->pb.human_cap * kHumanFloats, (size_t)n * kHumanFloats * sizeof(float));
    return n;
}
int b200pose_post_draw(b200pose_post* p, unsigned char* frames, int on_device, int n, const int* frame_hw,
                       const int* net_hw, void* cuda_stream) {
    if (!p) return fail("post_draw: null post");
    if (p->cur_ticket < 0) return fail("post_draw: no run selected (b200pose_post_select or b200pose_post_sync first)");
    if (n < 1 || n > p->pb.batch_cap) return fail("post_draw: n = %d images, must be 1 .. batch_cap %d", n, p->pb.batch_cap);
    if (n > p->slot_n[p->cur]) return fail("post_draw: n = %d images, the selected run has %d", n, p->slot_n[p->cur]);
    if (!frames || !frame_hw || !net_hw) return fail("post_draw: null frames, frame_hw or net_hw");
    for (int i = 0; i < n; ++i) {
        if (frame_hw[2 * i] < 1 || frame_hw[2 * i + 1] < 1)
            return fail("post_draw: frame_hw of image %d is %d x %d (sizes must be >= 1)", i, frame_hw[2 * i], frame_hw[2 * i + 1]);
        if (net_hw[2 * i] < 1 || net_hw[2 * i + 1] < 1)
            return fail("post_draw: net_hw of image %d is %d x %d (sizes must be >= 1)", i, net_hw[2 * i], net_hw[2 * i + 1]);
    }
    CU(cudaSetDevice(p->device));
    cudaStream_t st = (cudaStream_t)cuda_stream;
    // job: images [n] | person_img [P] | rows [P][73], each part 16-byte aligned
    const float* slot = p->hp_humans[p->cur].p;
    std::vector<DrawImage> imgs(n);
    long long bytes = 0;
    int persons = 0, max_h = 0, max_w = 0;
    for (int i = 0; i < n; ++i) {
        const int h = frame_hw[2 * i], w = frame_hw[2 * i + 1];
        imgs[i] = DrawImage{h, w, net_hw[2 * i], net_hw[2 * i + 1], persons, p->hp_nh[p->cur].p[i], bytes};
        persons += imgs[i].persons;
        bytes += 3LL * h * w;
        max_h = h > max_h ? h : max_h;
        max_w = w > max_w ? w : max_w;
    }
    auto up16 = [](size_t v) { return (v + 15) & ~(size_t)15; };
    const size_t o_pimg = up16(n * sizeof(DrawImage)), o_rows = o_pimg + up16(persons * sizeof(int));
    std::vector<char> job(o_rows + (size_t)persons * kHumanFloats * sizeof(float));
    memcpy(job.data(), imgs.data(), n * sizeof(DrawImage));
    for (int i = 0; i < n; ++i)
        for (int k = 0; k < imgs[i].persons; ++k) {
            const int q = imgs[i].person0 + k;
            reinterpret_cast<int*>(job.data() + o_pimg)[q] = i;
            memcpy(job.data() + o_rows + (size_t)q * kHumanFloats * sizeof(float),
                   slot + ((size_t)i * p->pb.human_cap + k) * kHumanFloats, kHumanFloats * sizeof(float));
        }
    if (persons == 0) return 0;      // nothing to draw: the frames stay as they are
    // the previous draw may still read the job, primitive and staging buffers (on another stream)
    if (p->have_draw) {
        if (job.size() > p->draw_job.n || (size_t)persons * kDrawPrimsPerPerson > p->draw_prims.n ||
            (!on_device && (size_t)bytes > p->draw_frames.n))
            CU(cudaEventSynchronize(p->ev_draw));
        CU(cudaStreamWaitEvent(st, p->ev_draw, 0));
    }
    CU(p->draw_job.ensure(job.size()));
    CU(p->draw_prims.ensure((size_t)persons * kDrawPrimsPerPerson));
    CU(cudaMemcpyAsync(p->draw_job.p, job.data(), job.size(), cudaMemcpyHostToDevice, st));
    unsigned char* d_frames = frames;
    if (!on_device) {
        CU(p->draw_frames.ensure((size_t)bytes));
        d_frames = p->draw_frames.p;
        CU(cudaMemcpyAsync(d_frames, frames, (size_t)bytes, cudaMemcpyHostToDevice, st));
    }
    const char* d = p->draw_job.p;
    if (launched(draw_launch(reinterpret_cast<const DrawImage*>(d), n, reinterpret_cast<const float*>(d + o_rows),
                             reinterpret_cast<const int*>(d + o_pimg), persons, p->draw_prims.p, max_h, max_w, d_frames, st),
                 "draw_launch", 2))
        return 1;
    if (!on_device) CU(cudaMemcpyAsync(frames, d_frames, (size_t)bytes, cudaMemcpyDeviceToHost, st));
    CU(cudaEventRecord(p->ev_draw, st));
    p->have_draw = true;
    if (!on_device) CU(cudaStreamSynchronize(st));
    return 0;
}
int b200pose_post_get_peaks(b200pose_post* p, int img, float* out, int max_peaks) {
    // valid for the LATEST run only (reads the device peak arrays, which the next run overwrites)
    if (!p || p->runs == 0 || b200pose_post_select(p, p->runs - 1)) return -1;
    const int last_n = p->slot_n[p->cur];
    if (img < 0 || img >= last_n) return -1;
    const PostBuffers& pb = p->pb;
    const size_t per = (size_t)18 * pb.peak_cap;
    if (p->h_px.empty()) {
        const size_t tot = per * last_n;
        p->h_px.resize(tot); p->h_py.resize(tot); p->h_px_s.resize(tot);
        cudaError_t e = cudaMemcpy(p->h_px.data(), pb.peak_x, tot * 4, cudaMemcpyDeviceToHost);
        if (e == cudaSuccess) e = cudaMemcpy(p->h_py.data(), pb.peak_y, tot * 4, cudaMemcpyDeviceToHost);
        if (e == cudaSuccess) e = cudaMemcpy(p->h_px_s.data(), pb.peak_s, tot * 4, cudaMemcpyDeviceToHost);
        if (e != cudaSuccess) { cuda_fail("peak copy failed: %s", cudaGetErrorString(e)); return -1; }
    }
    int k = 0;
    for (int part = 0; part < 18; ++part) {
        const int c = p->hp_counts[p->cur].p[(size_t)img * 18 + part];
        for (int i = 0; i < c && k < max_peaks; ++i, ++k) {
            const size_t o = (size_t)img * per + (size_t)part * pb.peak_cap + i;
            out[5 * k + 0] = (float)p->h_px[o];
            out[5 * k + 1] = (float)p->h_py[o];
            out[5 * k + 2] = p->h_px_s[o];
            out[5 * k + 3] = (float)k;
            out[5 * k + 4] = (float)part;
        }
    }
    return k;
}

// ------------------------------------------------------------------------------------------------ flip TTA
static int flip_merge_dev(const float* nh, const float* fh, const float* np_, const float* fp, int layout, int n, int h,
                          int w, float* oh, float* op, cudaStream_t st, const int* ext = nullptr) {
    cudaError_t e;
    if (layout == 0) {
        e = tta_flip_merge(nh, fh, oh, n, kHeat, h, w, (long)h * w, w, 1, ext, st);
        if (e == cudaSuccess) e = tta_flip_merge(np_, fp, op, n, kPaf, h, w, (long)h * w, w, 1, ext, st);
    } else {
        e = tta_flip_merge(nh, fh, oh, n, kHeat, h, w, 1, (long)w * kHeat, kHeat, ext, st);
        if (e == cudaSuccess) e = tta_flip_merge(np_, fp, op, n, kPaf, h, w, 1, (long)w * kPaf, kPaf, ext, st);
    }
    return launched(e, "tta_flip_merge", 2);
}

int b200pose_flip_merge(b200pose_post* p, const float* normal_heat, const float* flipped_heat, const float* normal_paf,
                        const float* flipped_paf, int on_device, int layout, int n, int h, int w, float* out_heat,
                        float* out_paf, void* cuda_stream) {
    if (!p) return fail("null post");
    if (n < 1 || h < 1 || w < 1 || (layout != 0 && layout != 1)) return fail("flip_merge: bad shape / layout");
    if (!normal_heat || !flipped_heat || !normal_paf || !flipped_paf || !out_heat || !out_paf) return fail("flip_merge: null pointer");
    CU(cudaSetDevice(p->device));
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (on_device)
        return flip_merge_dev(normal_heat, flipped_heat, normal_paf, flipped_paf, layout, n, h, w, out_heat, out_paf, st);
    const size_t eh = (size_t)n * kHeat * h * w, ep = (size_t)n * kPaf * h * w;
    CU(p->tta_in.ensure(2 * (eh + ep)));
    CU(p->tta_out.ensure(eh + ep));
    float *d_nh = p->tta_in.p, *d_fh = d_nh + eh, *d_np = d_fh + eh, *d_fp = d_np + ep;
    float *d_oh = p->tta_out.p, *d_op = d_oh + eh;
    CU(cudaMemcpyAsync(d_nh, normal_heat, eh * 4, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(d_fh, flipped_heat, eh * 4, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(d_np, normal_paf, ep * 4, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(d_fp, flipped_paf, ep * 4, cudaMemcpyHostToDevice, st));
    if (int rc = flip_merge_dev(d_nh, d_fh, d_np, d_fp, layout, n, h, w, d_oh, d_op, st)) return rc;
    CU(cudaMemcpyAsync(out_heat, d_oh, eh * 4, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(out_paf, d_op, ep * 4, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    return 0;
}

// ------------------------------------------------------------------------------------------------ fused inference
// Every fused entry point checks its handles, stages its frames (with their mirror images when flip), runs the
// forward pass and finishes with finish_infer.

static int check_infer(const b200pose_net* net, const b200pose_post* post, int mode) {
    if (!net || !post) return fail("null handle");
    if (!net->finalized) return fail("net not finalized");
    if (net->device != post->device) return fail("net and post live on different devices");
    return check_mode(net, mode);
}

// fp16: behind a fused run's forward of nimg images, copies the net's overflow flags into the next row of the run's slot
// (b200pose_post_overflow reads them once the run is fetched).  Stream-ordered before the run's post-processing, whose
// completion the fetch waits for.
static int stash_overflow(const b200pose_net* net, b200pose_post* post, int nimg, cudaStream_t st) {
    if (net->last.fp32 || tc_aux(net->last.fmt) != TcAux::kOverflow) return 0;
    if (post->ovf_pending >= kMaxOvfRows || nimg > 2 * post->pb.batch_cap) return fail("overflow rows exhausted");
    unsigned* dst = post->hp_ovf[post->runs & 1].p + (size_t)post->ovf_pending * 2 * post->pb.batch_cap;
    CU(cudaMemcpyAsync(dst, net->ovf.p, nimg * sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    post->ovf_pending += 1;
    post->ovf_pending_imgs = nimg;
    return 0;
}

// Flip TTA: merges the last forward's 2n images [frames | mirrors] of final maps into n maps at oh / op.
static int merge_last_flip(const b200pose_net* net, int n, float* oh, float* op, cudaStream_t st) {
    const int h = net->last.H / 8, w = net->last.W / 8;
    const size_t eh = (size_t)n * kHeat * h * w, ep = (size_t)n * kPaf * h * w;
    const float *heat = last_heat(net), *paf = last_paf(net);
    return flip_merge_dev(heat, heat + eh, paf, paf + ep, 0, n, h, w, oh, op, st, net->last.ext);
}

// Post-processing of the n frames of the last forward (flip: merged from its 2n images into post->d_heat / d_paf).
static int finish_infer(const b200pose_net* net, b200pose_post* post, int n, int flip, float thresh, cudaStream_t st) {
    const int h = net->last.H / 8, w = net->last.W / 8;
    const float *heat = last_heat(net), *paf = last_paf(net);
    if (flip) {
        CU(post->d_heat.ensure((size_t)n * kHeat * h * w));
        CU(post->d_paf.ensure((size_t)n * kPaf * h * w));
        if (int rc = merge_last_flip(net, n, post->d_heat.p, post->d_paf.p, st)) return rc;
        heat = post->d_heat.p;
        paf = post->d_paf.p;
    }
    return post_run_dev(post, heat, paf, 0, n, h, w, thresh, st, net->last.ext);
}

static int infer_impl(b200pose_net* net, b200pose_post* post, const void* input, int in_u8, int input_on_device, int n,
                      int H, int W, int mode, float thresh, int flip, void* cuda_stream) {
    if (int rc = check_infer(net, post, mode)) return rc;
    if (n < 1 || H < 8 || W < 8 || (H % 8) || (W % 8)) return fail("input must be [n,3,H,W] with H, W multiples of 8");
    if (int rc = check_batch(post, n)) return rc;
    post->ovf_pending = 0;
    post->jpeg_pending = 0;
    post->png_pending = 0;
    CU(cudaSetDevice(net->device));
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (flip) {   // the 2n batch [frames | mirrored frames] is assembled in the net's staging buffer
        const size_t elems = (size_t)n * 3 * H * W;
        const cudaMemcpyKind kind = input_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
        cudaError_t e;
        if (in_u8) {
            CU(net->in_stage_u8.ensure(2 * elems));
            CU(cudaMemcpyAsync(net->in_stage_u8.p, input, elems, kind, st));
            std::vector<RaggedFrame> tab(n);       // already cropped frames: the geometry is unused
            for (int i = 0; i < n; ++i) tab[i] = RaggedFrame{(long long)i * H * W * 3, H, W, CropGeom{}};
            if (int rc = upload_frames(net, tab, st)) return rc;
            e = tta_mirror_frames(net->in_stage_u8.p, net->in_stage_u8.p + elems, net->d_frames.p, n, (long)H * W * 3, st);
            input = net->in_stage_u8.p;
        } else {
            CU(net->in_stage.ensure(2 * elems));
            CU(cudaMemcpyAsync(net->in_stage.p, input, elems * 4, kind, st));
            e = tta_mirror_f32(net->in_stage.p, net->in_stage.p + elems, (long)n * 3, H, W, st);
            input = net->in_stage.p;
        }
        if (launched(e, "tta_mirror")) return 1;
        input_on_device = 1;
    }
    // host input is staged asynchronously: the caller keeps it alive until b200pose_post_sync()
    if (int rc = net_forward_impl(net, input, in_u8, input_on_device, flip ? 2 * n : n, H, W, mode, nullptr, 1, st, false))
        return rc;
    if (int rc = stash_overflow(net, post, flip ? 2 * n : n, st)) return rc;
    return finish_infer(net, post, n, flip, thresh, st);
}

int b200pose_infer(b200pose_net* net, b200pose_post* post, const float* input, int input_on_device, int n, int H, int W,
                   int mode, float thresh, void* cuda_stream) {
    return infer_impl(net, post, input, 0, input_on_device, n, H, W, mode, thresh, 0, cuda_stream);
}
int b200pose_infer_u8(b200pose_net* net, b200pose_post* post, const unsigned char* images, int input_on_device, int n,
                      int H, int W, int mode, float thresh, void* cuda_stream) {
    return infer_impl(net, post, images, 1, input_on_device, n, H, W, mode, thresh, 0, cuda_stream);
}
int b200pose_infer_flip(b200pose_net* net, b200pose_post* post, const float* input, int input_on_device, int n, int H,
                        int W, int mode, float thresh, void* cuda_stream) {
    return infer_impl(net, post, input, 0, input_on_device, n, H, W, mode, thresh, 1, cuda_stream);
}
int b200pose_infer_u8_flip(b200pose_net* net, b200pose_post* post, const unsigned char* images, int input_on_device,
                           int n, int H, int W, int mode, float thresh, void* cuda_stream) {
    return infer_impl(net, post, images, 1, input_on_device, n, H, W, mode, thresh, 1, cuda_stream);
}

// ------------------------------------------------------------------------------------------------ crop_with_factor
static int crop_check(int n, int src_h, int src_w, int dest_size, int factor, CropGeom* g) {
    if (n < 1 || src_h < 1 || src_w < 1 || dest_size < 1) return fail("crop_with_factor: bad shape");
    if (n > 65535) return fail("crop_with_factor: %d images (at most 65535)", n);
    if (factor < 8 || factor % 8) return fail("crop_with_factor: factor must be a multiple of 8 (the network's stride)");
    *g = crop_geometry(src_h, src_w, dest_size, factor);
    if (g->res_h < 1 || g->res_w < 1) return fail("crop_with_factor: the resized frame would be empty");
    if ((long)g->pad_h * g->pad_w > (1L << 28)) return fail("crop_with_factor: resized frame too large");
    return 0;
}

int b200pose_crop_geometry(int src_h, int src_w, int dest_size, int factor, double* im_scale, int* res_h, int* res_w,
                           int* pad_h, int* pad_w) {
    CropGeom g;
    if (int rc = crop_check(1, src_h, src_w, dest_size, factor, &g)) return rc;
    if (im_scale) *im_scale = g.im_scale;
    if (res_h) *res_h = g.res_h;
    if (res_w) *res_w = g.res_w;
    if (pad_h) *pad_h = g.pad_h;
    if (pad_w) *pad_w = g.pad_w;
    return 0;
}

int b200pose_net_crop_with_factor(b200pose_net* net, const unsigned char* images, int images_on_device, int n, int src_h,
                                  int src_w, int dest_size, int factor, unsigned char* out, int out_on_device,
                                  void* cuda_stream) {
    if (!net) return fail("null net");
    if (!images || !out) return fail("crop_with_factor: null pointer");
    CropGeom g;
    if (int rc = crop_check(n, src_h, src_w, dest_size, factor, &g)) return rc;
    CU(cudaSetDevice(net->device));
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    const size_t raw = (size_t)n * src_h * src_w * 3, outb = (size_t)n * g.pad_h * g.pad_w * 3;
    const unsigned char* d_in;
    if (int rc = stage_raw(net, images, images_on_device, raw, 0, st, &d_in)) return rc;
    unsigned char* d_out = out;
    if (!out_on_device) {
        CU(net->in_stage_u8.ensure(outb));
        d_out = net->in_stage_u8.p;
    }
    std::vector<RaggedFrame> tab(n);
    for (int i = 0; i < n; ++i) tab[i] = RaggedFrame{(long long)i * src_h * src_w * 3, src_h, src_w, g};
    if (int rc = upload_frames(net, tab, st)) return rc;
    if (launched(crop_frames_launch(d_in, net->d_frames.p, n, d_out, g.pad_h, g.pad_w, st), "crop_frames_launch")) return 1;
    if (!out_on_device) CU(cudaMemcpyAsync(out, d_out, outb, cudaMemcpyDeviceToHost, st));
    if (!images_on_device || !out_on_device) CU(cudaStreamSynchronize(st));
    return 0;
}

// n raw frames of one size src_h x src_w (src_hw null) or of the sizes src_hw[2 i], src_hw[2 i + 1] (a ragged batch),
// cropped for dest_size.
static int raw_batch(int n, int src_h, int src_w, const int* src_hw, int dest_size, int factor, int flip, RawBatch* c) {
    const int nimg = flip ? 2 * n : n;
    if (src_hw && nimg > kMaxRagged) return fail("ragged batch: %d images (at most %d)", nimg, kMaxRagged);
    *c = RawBatch{};
    c->tab.assign(nimg, RaggedFrame{});
    for (int i = 0; i < n; ++i) {
        RaggedFrame& f = c->tab[i];
        f.src_h = src_hw ? src_hw[2 * i] : src_h;
        f.src_w = src_hw ? src_hw[2 * i + 1] : src_w;
        if (int rc = crop_check(1, f.src_h, f.src_w, dest_size, factor, &f.g)) return rc;
        f.off = c->raw;
        const long long b = (long long)f.src_h * f.src_w * 3;
        c->raw += b;
        if (b > c->max_bytes) c->max_bytes = b;
        if (f.g.pad_h > c->Hc) c->Hc = f.g.pad_h;
        if (f.g.pad_w > c->Wc) c->Wc = f.g.pad_w;
    }
    for (int i = 0; i < n && flip; ++i) {      // mirrored raw frames follow the originals in the staging buffer
        c->tab[n + i] = c->tab[i];
        c->tab[n + i].off += c->raw;
    }
    for (int i = 0; i < nimg && src_hw; ++i) {
        c->ext.push_back(c->tab[i].g.pad_h);
        c->ext.push_back(c->tab[i].g.pad_w);
    }
    if ((long)c->Hc * c->Wc > (1L << 28)) return fail("infer_raw: canvas too large");
    return 0;
}

// ------------------------------------------------------------------------------------------------ video frames
// The frames of one b200pose_net_convert_frames / b200pose_infer_frames call, checked: the source table
// convert_frames_kernel reads (host planes until they are staged), the rotated sizes [oh_0, ow_0, oh_1, ...], the packed
// BGR output's size and the largest rotated frame's pixel count.
struct FrameBatch {
    std::vector<FrameSrc> tab;
    std::vector<int> hw;
    int format = 0, rotate = 0;
    long long bytes = 0, max_px = 0;
    bool uniform() const {
        for (size_t i = 2; i < hw.size(); i += 2)
            if (hw[i] != hw[0] || hw[i + 1] != hw[1]) return false;
        return true;
    }
};

constexpr const char* kFrameFormatName[3] = {"BGR", "NV12", "I420"};

// Plane k of a stored h x w frame of `format`: bytes per row and rows.
static void frame_plane_shape(int format, int k, int h, int w, long* row, int* rows) {
    *row = format == kFrameBGR ? 3L * w : (k == 0 || format == kFrameNV12 ? (long)w : (long)w / 2);
    *rows = k == 0 ? h : h / 2;
}

static int frame_planes(int format) { return format == kFrameBGR ? 1 : (format == kFrameNV12 ? 2 : 3); }

// Checks every frame of a call before anything is enqueued.
static int check_frames(const b200pose_frame* frames, int n, int max_n, int format, int rotate, FrameBatch* b) {
    if (format < kFrameBGR || format > kFrameI420)
        return fail("frames: format %d is unknown (B200POSE_FRAME_BGR 0, _NV12 1, _I420 2)", format);
    if (rotate != 0 && rotate != 90 && rotate != 180 && rotate != 270)
        return fail("frames: rotate %d (0, 90, 180 or 270 degrees clockwise)", rotate);
    if (!frames) return fail("frames: null frame table");
    if (n < 1 || n > max_n) return fail("frames: %d frames (1 .. %d)", n, max_n);
    *b = FrameBatch{};
    b->format = format;
    b->rotate = rotate;
    for (int i = 0; i < n; ++i) {
        const b200pose_frame& f = frames[i];
        if (f.h < 1 || f.w < 1 || (long)f.h * f.w > (1L << 28))
            return fail("frame %d: size h = %d, w = %d (1 .. 2^28 pixels)", i, f.h, f.w);
        if (format != kFrameBGR && (f.h % 2 || f.w % 2))
            return fail("frame %d: %s needs even sizes, h = %d, w = %d", i, kFrameFormatName[format], f.h, f.w);
        FrameSrc s{};
        for (int k = 0; k < frame_planes(format); ++k) {
            long row;
            int rows;
            frame_plane_shape(format, k, f.h, f.w, &row, &rows);
            if (!f.plane[k]) return fail("frame %d: plane[%d] is null", i, k);
            if (f.pitch[k] < row)
                return fail("frame %d: pitch[%d] = %d is shorter than a %s row of %ld bytes", i, k, f.pitch[k],
                            kFrameFormatName[format], row);
            s.plane[k] = f.plane[k];
            s.pitch[k] = f.pitch[k];
        }
        s.h = f.h;
        s.w = f.w;
        s.off = b->bytes;
        int oh, ow;
        fr_rotated_size(f.h, f.w, rotate, &oh, &ow);
        b->hw.push_back(oh);
        b->hw.push_back(ow);
        b->bytes += (long long)oh * ow * 3;
        if ((long long)oh * ow > b->max_px) b->max_px = (long long)oh * ow;
        b->tab.push_back(s);
    }
    return 0;
}

// Packed BGR frames (pitch 3w, frame i + 1 right behind frame i) that need no rotation: the raw-frame path reads them
// as they are.
static bool frames_are_packed_bgr(const FrameBatch& b) {
    if (b.format != kFrameBGR || b.rotate != 0) return false;
    for (const FrameSrc& s : b.tab)
        if (s.pitch[0] != 3 * s.w || s.plane[0] != b.tab[0].plane[0] + s.off) return false;
    return true;
}

// Converts the frames of b into `out` (device, b.bytes): host planes are first copied, packed, into net->frame_stage.
static int convert_frames_dev(b200pose_net* net, const FrameBatch& b, int on_device, unsigned char* out, cudaStream_t st) {
    std::vector<FrameSrc> tab = b.tab;
    const int planes = frame_planes(b.format);
    if (!on_device) {
        size_t total = 0;
        for (const FrameSrc& s : tab)
            for (int k = 0; k < planes; ++k) {
                long row;
                int rows;
                frame_plane_shape(b.format, k, s.h, s.w, &row, &rows);
                total += (size_t)row * rows;
            }
        CU(net->frame_stage.ensure(total));
        size_t at = 0;
        for (FrameSrc& s : tab)
            for (int k = 0; k < planes; ++k) {
                long row;
                int rows;
                frame_plane_shape(b.format, k, s.h, s.w, &row, &rows);
                CU(cudaMemcpy2DAsync(net->frame_stage.p + at, row, s.plane[k], s.pitch[k], row, rows,
                                     cudaMemcpyHostToDevice, st));
                s.plane[k] = net->frame_stage.p + at;
                s.pitch[k] = (int)row;
                at += (size_t)row * rows;
            }
    }
    CU(net->d_frame_src.ensure(tab.size()));
    CU(cudaMemcpyAsync(net->d_frame_src.p, tab.data(), tab.size() * sizeof(FrameSrc), cudaMemcpyHostToDevice, st));
    return launched(convert_frames_launch(net->d_frame_src.p, (int)tab.size(), b.format, b.rotate, (long)b.max_px, out, st),
                    "convert_frames_launch");
}

// The frames of b converted into net->raw_stage, with room for their mirror images behind them when flip: what
// stage_raw makes of packed BGR frames.
static int stage_frames(b200pose_net* net, const FrameBatch& b, int on_device, int flip, cudaStream_t st,
                        const unsigned char** d_raw) {
    CU(net->raw_stage.ensure((size_t)b.bytes * (flip ? 2 : 1)));
    *d_raw = net->raw_stage.p;
    return convert_frames_dev(net, b, on_device, net->raw_stage.p, st);
}

// ------------------------------------------------------------------------------------------------ JPEG streams
constexpr long long kJpegMaxPixels = 1LL << 28;     // a frame's pixels, as for video frames

// The streams of one b200pose_net_decode_jpegs / b200pose_infer_jpegs call, parsed and checked: the upload image and
// where its tables lie, the oriented sizes [oh_0, ow_0, oh_1, ...], the packed BGR output's size, and what the device
// buffers must hold.
struct JpegCall {
    int n = 0, nwork = 0, njobs = 0, nprog = 0;
    std::vector<char> up;
    size_t o_ims = 0, o_jobs = 0, o_segs = 0, o_chunk = 0, o_work = 0, o_status = 0, o_raw = 0, o_prog = 0, o_scans = 0,
           o_pseg = 0;
    std::vector<int> hw;
    long long bytes = 0, data = 0, blocks = 0, planes = 0, max_blocks = 0, max_px = 0;
    bool uniform() const {
        for (size_t i = 2; i < hw.size(); i += 2)
            if (hw[i] != hw[0] || hw[i + 1] != hw[1]) return false;
        return true;
    }
};

// Parses every stream of a call before anything is enqueued and lays out its upload.  progressive: progressive
// streams are decoded too (b200pose_net_set_jpeg_progressive); each of their scans is an unstuffing job of its own.
static int check_jpegs(const unsigned char* const* data, const long long* sizes, int n, int max_n, JpegCall* j,
                       bool progressive) {
    if (!data || !sizes) return fail("jpegs: null stream table");
    if (n < 1 || n > max_n) return fail("jpegs: %d images (1 .. %d)", n, max_n);
    *j = JpegCall{};
    j->n = n;
    std::unique_ptr<JpegParsed> P(new JpegParsed);
    std::vector<JpegImage> ims(n);
    std::vector<JpegUnstuffJob> jobs;
    std::vector<JpegSeg> segs, psegs;
    std::vector<JpegProgImage> progs;
    std::vector<JpegScan> pscans;
    std::vector<unsigned> status(n);
    std::vector<std::pair<long long, long long>> scans;      // per job, its bytes of the stream
    std::vector<int> job_img;
    long long raw = 0, chunks = 0;
    for (int i = 0; i < n; ++i) {
        if (!data[i] || sizes[i] < 0) return fail("jpeg image %d: null stream or negative size", i);
        if (!jpeg_parse(data[i], sizes[i], kJpegMaxPixels, P.get(), progressive)) return fail("jpeg image %d: %s", i, P->reason);
        if (!P->supported) return fail("jpeg image %d: %s", i, P->reason);
        JpegImage& im = ims[i];
        im = P->im;
        im.out = j->bytes;
        for (int c = 0; c < im.ncomp; ++c) {
            JpegComp& cp = im.comp[c];
            cp.coef = j->blocks;
            cp.plane = j->planes;
            j->blocks += (long long)cp.bw * cp.bh;
            j->planes += (long long)cp.bw * cp.bh * 64;
            j->max_blocks = std::max(j->max_blocks, (long long)cp.bw * cp.bh);
        }
        j->hw.push_back(im.oh);
        j->hw.push_back(im.ow);
        j->bytes += 3LL * im.oh * im.ow;
        j->max_px = std::max(j->max_px, (long long)im.oh * im.ow);
        status[i] = P->status;
        if (P->progressive) {      // each scan's unstuffed data gets room for its raw bytes
            std::vector<long long> base;
            for (size_t s = 0; s < P->scans.size(); ++s) {
                const long long b = P->scan_raw[2 * s], e = P->scan_raw[2 * s + 1];
                jobs.push_back(JpegUnstuffJob{raw, raw + (e - b), j->data});
                scans.push_back({b, e});
                job_img.push_back(i);
                base.push_back(j->data);
                j->data += e - b;
                raw += e - b;
            }
            progs.push_back(JpegProgImage{i, (int)pscans.size(), (int)P->scans.size()});
            jpeg_prog_segments(*P, i, base.data(), &pscans, &psegs);
            continue;
        }
        jobs.push_back(JpegUnstuffJob{raw, raw + (P->scan_end - P->scan_beg), j->data});
        scans.push_back({P->scan_beg, P->scan_end});
        job_img.push_back(i);
        chunks += jpeg_segments(*P, i, j->data, chunks, &segs);
        j->data += P->seg_end.back();
        raw += P->scan_end - P->scan_beg;
    }
    std::vector<int> chunk_seg;
    std::vector<long long> work;
    jpeg_work(segs, chunks, &chunk_seg, &work);
    j->nwork = (int)work.size() - 1;
    j->njobs = (int)jobs.size();
    j->nprog = (int)progs.size();
    auto up16 = [](size_t v) { return (v + 15) & ~(size_t)15; };
    j->o_ims = 0;
    j->o_jobs = up16(j->o_ims + n * sizeof(JpegImage));
    j->o_segs = up16(j->o_jobs + jobs.size() * sizeof(JpegUnstuffJob));
    j->o_chunk = up16(j->o_segs + segs.size() * sizeof(JpegSeg));
    j->o_work = up16(j->o_chunk + chunk_seg.size() * sizeof(int));
    j->o_status = up16(j->o_work + work.size() * sizeof(long long));
    j->o_prog = up16(j->o_status + n * sizeof(unsigned));
    j->o_scans = up16(j->o_prog + progs.size() * sizeof(JpegProgImage));
    j->o_pseg = up16(j->o_scans + pscans.size() * sizeof(JpegScan));
    j->o_raw = up16(j->o_pseg + psegs.size() * sizeof(JpegSeg));
    j->up.resize(j->o_raw + (size_t)raw + 16);
    char* u = j->up.data();
    memcpy(u + j->o_ims, ims.data(), n * sizeof(JpegImage));
    memcpy(u + j->o_jobs, jobs.data(), jobs.size() * sizeof(JpegUnstuffJob));
    memcpy(u + j->o_segs, segs.data(), segs.size() * sizeof(JpegSeg));
    memcpy(u + j->o_chunk, chunk_seg.data(), chunk_seg.size() * sizeof(int));
    memcpy(u + j->o_work, work.data(), work.size() * sizeof(long long));
    memcpy(u + j->o_status, status.data(), n * sizeof(unsigned));
    memcpy(u + j->o_prog, progs.data(), progs.size() * sizeof(JpegProgImage));
    memcpy(u + j->o_scans, pscans.data(), pscans.size() * sizeof(JpegScan));
    memcpy(u + j->o_pseg, psegs.data(), psegs.size() * sizeof(JpegSeg));
    for (size_t k = 0; k < jobs.size(); ++k)
        memcpy(u + j->o_raw + jobs[k].raw_beg, data[job_img[k]] + scans[k].first, (size_t)(scans[k].second - scans[k].first));
    return 0;
}

// Uploads the call's tables and scans in one copy and decodes the frames into `out` (device, j.bytes); the status
// words are at the returned device address.
static int decode_jpegs_dev(b200pose_net* net, const JpegCall& j, unsigned char* out, cudaStream_t st,
                            const unsigned** d_status) {
    CU(net->jpeg_in.ensure(j.up.size()));
    CU(net->jpeg_data.ensure((size_t)j.data + 16));
    CU(net->jpeg_coef.ensure((size_t)j.blocks * 64));
    CU(net->jpeg_planes.ensure((size_t)j.planes));
    CU(cudaMemcpyAsync(net->jpeg_in.p, j.up.data(), j.up.size(), cudaMemcpyHostToDevice, st));
    CU(cudaMemsetAsync(net->jpeg_coef.p, 0, (size_t)j.blocks * 64 * sizeof(short), st));
    char* d = net->jpeg_in.p;
    JpegBatch b;
    b.ims = reinterpret_cast<const JpegImage*>(d + j.o_ims);
    b.n = j.n;
    b.jobs = reinterpret_cast<const JpegUnstuffJob*>(d + j.o_jobs);
    b.raw = reinterpret_cast<const unsigned char*>(d + j.o_raw);
    b.data = net->jpeg_data.p;
    b.segs = reinterpret_cast<const JpegSeg*>(d + j.o_segs);
    b.chunk_seg = reinterpret_cast<const int*>(d + j.o_chunk);
    b.work = reinterpret_cast<const long long*>(d + j.o_work);
    b.nwork = j.nwork;
    b.coef = net->jpeg_coef.p;
    b.planes = net->jpeg_planes.p;
    b.out = out;
    b.status = reinterpret_cast<unsigned*>(d + j.o_status);
    b.max_blocks = j.max_blocks;
    b.max_px = j.max_px;
    b.njobs = j.njobs;
    b.prog = reinterpret_cast<const JpegProgImage*>(d + j.o_prog);
    b.nprog = j.nprog;
    b.scans = reinterpret_cast<const JpegScan*>(d + j.o_scans);
    b.pseg = reinterpret_cast<const JpegSeg*>(d + j.o_pseg);
    *d_status = b.status;
    return launched(jpeg_decode_launch(b, st), "jpeg_decode_launch", jpeg_decode_launches(b));
}

// The frames of j decoded into net->raw_stage, with room for their mirror images behind them when flip; the status
// words travel to the run's slot of the post object.
static int stage_jpegs(b200pose_net* net, b200pose_post* post, const JpegCall& j, int flip, cudaStream_t st,
                       const unsigned char** d_raw) {
    CU(net->raw_stage.ensure((size_t)j.bytes * (flip ? 2 : 1)));
    *d_raw = net->raw_stage.p;
    const unsigned* d_status;
    if (int rc = decode_jpegs_dev(net, j, net->raw_stage.p, st, &d_status)) return rc;
    CU(cudaMemcpyAsync(post->hp_jpeg[post->runs & 1].p, d_status, j.n * sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    post->jpeg_pending = j.n;
    return 0;
}

static const char* jpeg_status_name(unsigned s) {
    return s & kJpegBadCode ? "an invalid Huffman code" : s & kJpegShortData ? "the data ends before the last block"
         : s & kJpegExtraData ? "data left after the last block" : "missing or misordered restart markers";
}

// ------------------------------------------------------------------------------------------------ PNG streams
// The streams of one b200pose_net_decode_pngs / b200pose_infer_pngs call, parsed and checked: the upload image and
// where its tables lie, the oriented sizes [oh_0, ow_0, oh_1, ...], the packed BGR output's size, and what the device
// buffers must hold.
struct PngCall {
    int n = 0, nidat = 0;
    std::vector<char> up;
    size_t o_ims = 0, o_idat = 0, o_status = 0, o_raw = 0;
    std::vector<int> hw;
    long long bytes = 0, zlib = 0, rows = 0, max_px = 0;
    bool uniform() const {
        for (size_t i = 2; i < hw.size(); i += 2)
            if (hw[i] != hw[0] || hw[i + 1] != hw[1]) return false;
        return true;
    }
};

// Parses every stream of a call before anything is enqueued and lays out its upload: per image the bytes from its
// first IDAT chunk's type to its last one's data, which hold every IDAT chunk's type and data.
static int check_pngs(const unsigned char* const* data, const long long* sizes, int n, int max_n, PngCall* j) {
    if (!data || !sizes) return fail("pngs: null stream table");
    if (n < 1 || n > max_n) return fail("pngs: %d images (1 .. %d)", n, max_n);
    *j = PngCall{};
    j->n = n;
    std::unique_ptr<PngParsed> P(new PngParsed);
    std::vector<PngDecImage> ims(n);
    std::vector<PngIdat> idat;
    std::vector<std::pair<long long, long long>> spans(n);
    long long raw = 0;
    for (int i = 0; i < n; ++i) {
        if (!data[i] || sizes[i] < 0) return fail("png image %d: null stream or negative size", i);
        if (!png_parse(data[i], sizes[i], kJpegMaxPixels, P.get())) return fail("png image %d: %s", i, P->reason);
        if (!P->supported) return fail("png image %d: %s", i, P->reason);
        PngDecImage& im = ims[i];
        im = P->im;
        im.out = j->bytes;
        im.z0 = j->zlib;
        im.zlen = P->zlen;
        im.f0 = j->rows;
        im.idat0 = (int)idat.size();
        im.nidat = (int)P->idat.size();
        const long long beg = P->idat.front().src, end = P->idat.back().src + 4 + P->idat.back().len;
        for (PngIdat c : P->idat) {
            c.img = i;
            c.src += raw - beg;
            idat.push_back(c);
        }
        spans[i] = {beg, end};
        raw += end - beg;
        j->zlib += P->zlen;
        j->rows += im.flen;
        j->hw.push_back(im.oh);
        j->hw.push_back(im.ow);
        j->bytes += 3LL * im.oh * im.ow;
        j->max_px = std::max(j->max_px, (long long)im.oh * im.ow);
    }
    j->nidat = (int)idat.size();
    auto up16 = [](size_t v) { return (v + 15) & ~(size_t)15; };
    j->o_ims = 0;
    j->o_idat = up16(j->o_ims + n * sizeof(PngDecImage));
    j->o_status = up16(j->o_idat + idat.size() * sizeof(PngIdat));
    j->o_raw = up16(j->o_status + n * sizeof(unsigned));
    j->up.assign(j->o_raw + (size_t)raw + 16, 0);
    char* u = j->up.data();
    memcpy(u + j->o_ims, ims.data(), n * sizeof(PngDecImage));
    memcpy(u + j->o_idat, idat.data(), idat.size() * sizeof(PngIdat));
    for (long long at = 0, i = 0; i < n; at += spans[i].second - spans[i].first, ++i)
        memcpy(u + j->o_raw + at, data[i] + spans[i].first, (size_t)(spans[i].second - spans[i].first));
    return 0;
}

// Uploads the call's tables and chunks in one copy and decodes the frames into `out` (device, j.bytes); the status
// words are at the returned device address.
static int decode_pngs_dev(b200pose_net* net, const PngCall& j, unsigned char* out, cudaStream_t st,
                           const unsigned** d_status) {
    CU(net->png_in.ensure(j.up.size()));
    CU(net->png_zlib.ensure((size_t)j.zlib + 16));
    CU(net->png_rows.ensure((size_t)j.rows + 16));
    CU(cudaMemcpyAsync(net->png_in.p, j.up.data(), j.up.size(), cudaMemcpyHostToDevice, st));
    char* d = net->png_in.p;
    PngDecBatch b;
    b.ims = reinterpret_cast<const PngDecImage*>(d + j.o_ims);
    b.n = j.n;
    b.idat = reinterpret_cast<const PngIdat*>(d + j.o_idat);
    b.nidat = j.nidat;
    b.raw = reinterpret_cast<const unsigned char*>(d + j.o_raw);
    b.zlib = net->png_zlib.p;
    b.rows = net->png_rows.p;
    b.out = out;
    b.status = reinterpret_cast<unsigned*>(d + j.o_status);
    b.max_px = j.max_px;
    *d_status = b.status;
    return launched(png_decode_launch(b, st), "png_decode_launch", kPngLaunches);
}

// The frames of j decoded into net->raw_stage, with room for their mirror images behind them when flip; the status
// words travel to the run's slot of the post object.
static int stage_pngs(b200pose_net* net, b200pose_post* post, const PngCall& j, int flip, cudaStream_t st,
                      const unsigned char** d_raw) {
    CU(net->raw_stage.ensure((size_t)j.bytes * (flip ? 2 : 1)));
    *d_raw = net->raw_stage.p;
    const unsigned* d_status;
    if (int rc = decode_pngs_dev(net, j, net->raw_stage.p, st, &d_status)) return rc;
    CU(cudaMemcpyAsync(post->hp_png[post->runs & 1].p, d_status, j.n * sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    post->png_pending = j.n;
    return 0;
}

static const char* png_status_name(unsigned s) {
    return s & kPngBadCrc ? "a CRC error in an IDAT chunk" : s & kPngBadDeflate ? "invalid deflate data"
         : s & kPngShortData ? "the image data ends early" : s & kPngBadAdler ? "an Adler-32 mismatch"
         : "an invalid filter type";
}

// The fused inference of raw uint8 frames (b200pose_infer_raw_u8*): n frames of one size src_h x src_w, or of the
// sizes src_hw (a ragged batch), are staged with their mirror images when flip, cropped for every scale and run
// through the network.  scales null: one scale, base_size, post-processed as it is.  Else every scale s runs at
// int(base_size * s) and its maps are resized (bicubic) to the grid of base_size, averaged and post-processed.
// fb (b200pose_infer_frames): the frames are those of fb, converted into the staging buffer, instead of `images`;
// jb (b200pose_infer_jpegs): those of the JPEG streams of jb, decoded into the staging buffer; pc
// (b200pose_infer_pngs): those of the PNG streams of pc.
static int infer_raw(b200pose_net* net, b200pose_post* post, const unsigned char* images, int on_device, int n,
                     int src_h, int src_w, const int* src_hw, int base_size, int factor, const double* scales,
                     int n_scales, int mode, float thresh, int flip, void* cuda_stream, const FrameBatch* fb = nullptr,
                     const JpegCall* jb = nullptr, const PngCall* pc = nullptr) {
    if (int rc = check_infer(net, post, mode)) return rc;
    if (!images && !fb && !jb && !pc) return fail("infer_raw: null pointer");
    if (scales && (n_scales < 1 || n_scales > 16)) return fail("infer_raw: %d scales (1 .. 16)", n_scales);
    if (n < 1 || n > post->pb.batch_cap) return fail("batch %d outside 1 .. post batch_cap %d", n, post->pb.batch_cap);
    const bool ragged = src_hw != nullptr;
    post->ovf_pending = 0;
    post->jpeg_pending = 0;
    post->png_pending = 0;
    // every scale's geometry first: an invalid frame size fails before anything is enqueued
    RawBatch base;
    if (scales && raw_batch(n, src_h, src_w, src_hw, base_size, factor, 0, &base)) return 1;
    std::vector<RawBatch> sc(scales ? n_scales : 1);
    std::vector<RaggedResize> rz;
    for (int k = 0; k < (int)sc.size(); ++k) {
        const int dest = scales ? (int)((double)base_size * scales[k]) : base_size;       // Python: int(base_size * s)
        if (int rc = raw_batch(n, src_h, src_w, src_hw, dest, factor, flip, &sc[k])) return rc;
        for (int i = 0; i < n && scales; ++i) {
            const CropGeom &g = sc[k].tab[i].g, &g1 = base.tab[i].g;
            rz.push_back(ragged_resize(g.pad_h / 8, g.pad_w / 8, g1.pad_h / 8, g1.pad_w / 8));
        }
    }
    CU(cudaSetDevice(net->device));
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    // the caller keeps a host input alive until b200pose_post_sync(), as for b200pose_infer
    const unsigned char* d_raw;
    if (int rc = fb ? stage_frames(net, *fb, on_device, flip, st, &d_raw)
                 : jb ? stage_jpegs(net, post, *jb, flip, st, &d_raw)
                 : pc ? stage_pngs(net, post, *pc, flip, st, &d_raw)
                      : stage_raw(net, images, on_device, (size_t)sc[0].raw, flip, st, &d_raw))
        return rc;
    // the sources and offsets of the frame table are those of every scale
    if (upload_frames(net, sc[0].tab, st)) return 1;
    if (flip) {      // mirrored RAW frames, so that the padding of both orientations ends up on the right, as for the reference
        unsigned char* mirror = net->raw_stage.p + sc[0].raw;
        if (launched(tta_mirror_frames(net->raw_stage.p, mirror, net->d_frames.p, n, (long)sc[0].max_bytes, st), "tta_mirror"))
            return 1;
    }
    const int nimg = flip ? 2 * n : n;
    if (!scales) {
        if (int rc = crop_and_forward(net, d_raw, nimg, sc[0], mode, st)) return rc;
        if (int rc = stash_overflow(net, post, nimg, st)) return rc;
        return finish_infer(net, post, n, flip, thresh, st);
    }
    if (ragged) {
        CU(post->ms_ext.ensure(base.ext.size()));
        CU(cudaMemcpyAsync(post->ms_ext.p, base.ext.data(), base.ext.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    }
    CU(post->ms_resize.ensure(rz.size()));
    CU(cudaMemcpyAsync(post->ms_resize.p, rz.data(), rz.size() * sizeof(RaggedResize), cudaMemcpyHostToDevice, st));
    const int h1 = base.Hc / 8, w1 = base.Wc / 8;
    CU(post->d_heat.ensure((size_t)n * kHeat * h1 * w1));
    CU(post->d_paf.ensure((size_t)n * kPaf * h1 * w1));
    for (int k = 0; k < n_scales; ++k) {
        const RawBatch& c = sc[k];
        if (k > 0 && upload_frames(net, c.tab, st)) return 1;
        if (int rc = crop_and_forward(net, d_raw, nimg, c, mode, st)) return rc;
        if (int rc = stash_overflow(net, post, nimg, st)) return rc;
        const int h = c.Hc / 8, w = c.Wc / 8;
        const size_t eh = (size_t)n * kHeat * h * w, ep = (size_t)n * kPaf * h * w;
        const float *s_heat = last_heat(net), *s_paf = last_paf(net);
        if (flip) {
            CU(post->tta_out.ensure(eh + ep));
            if (int rc = merge_last_flip(net, n, post->tta_out.p, post->tta_out.p + eh, st)) return rc;
            s_heat = post->tta_out.p;
            s_paf = post->tta_out.p + eh;
        }
        const float div = (k == n_scales - 1) ? (float)n_scales : 0.f;
        const RaggedResize* f = post->ms_resize.p + (size_t)k * n;
        cudaError_t e = resize_cubic_accum_launch(s_heat, post->d_heat.p, f, n, kHeat, h, w, h1, w1, k == 0, div, st);
        if (e == cudaSuccess) e = resize_cubic_accum_launch(s_paf, post->d_paf.p, f, n, kPaf, h, w, h1, w1, k == 0, div, st);
        if (launched(e, "resize_cubic_accum", 2)) return 1;
    }
    // the net's extents table now holds the last scale's: post-processing reads the base extents
    return post_run_dev(post, post->d_heat.p, post->d_paf.p, 0, n, h1, w1, thresh, st, ragged ? post->ms_ext.p : nullptr);
}

int b200pose_infer_raw_u8(b200pose_net* net, b200pose_post* post, const unsigned char* images, int input_on_device, int n,
                          int src_h, int src_w, int dest_size, int factor, int mode, float thresh, int flip,
                          void* cuda_stream) {
    return infer_raw(net, post, images, input_on_device, n, src_h, src_w, nullptr, dest_size, factor, nullptr, 0, mode,
                     thresh, flip, cuda_stream);
}

int b200pose_infer_raw_u8_ragged(b200pose_net* net, b200pose_post* post, const unsigned char* images, int input_on_device,
                                  int n, const int* src_hw, int dest_size, int factor, int mode, float thresh, int flip,
                                  void* cuda_stream) {
    return src_hw ? infer_raw(net, post, images, input_on_device, n, 0, 0, src_hw, dest_size, factor, nullptr, 0, mode,
                              thresh, flip, cuda_stream)
                  : fail("infer_raw_ragged: null size table");
}

int b200pose_infer_raw_u8_multiscale(b200pose_net* net, b200pose_post* post, const unsigned char* images,
                                     int input_on_device, int n, int src_h, int src_w, int base_size, int factor,
                                     const double* scales, int n_scales, int mode, float thresh, int flip,
                                     void* cuda_stream) {
    return scales ? infer_raw(net, post, images, input_on_device, n, src_h, src_w, nullptr, base_size, factor, scales,
                              n_scales, mode, thresh, flip, cuda_stream)
                  : fail("infer_multiscale: null scales");
}

int b200pose_infer_raw_u8_multiscale_ragged(b200pose_net* net, b200pose_post* post, const unsigned char* images,
                                            int input_on_device, int n, const int* src_hw, int base_size, int factor,
                                            const double* scales, int n_scales, int mode, float thresh, int flip,
                                            void* cuda_stream) {
    return scales && src_hw ? infer_raw(net, post, images, input_on_device, n, 0, 0, src_hw, base_size, factor, scales,
                                        n_scales, mode, thresh, flip, cuda_stream)
                            : fail("infer_multiscale_ragged: null pointer");
}

int b200pose_net_convert_frames(b200pose_net* net, const b200pose_frame* frames, int n, int format, int on_device,
                                int rotate, unsigned char* out, int out_on_device, void* cuda_stream) {
    if (!net) return fail("null net");
    if (!out) return fail("convert_frames: null output");
    FrameBatch b;
    if (int rc = check_frames(frames, n, kMaxRagged, format, rotate, &b)) return rc;
    CU(cudaSetDevice(net->device));
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    unsigned char* d_out = out;
    if (!out_on_device) {
        CU(net->raw_stage.ensure((size_t)b.bytes));
        d_out = net->raw_stage.p;
    }
    if (int rc = convert_frames_dev(net, b, on_device, d_out, st)) return rc;
    if (!out_on_device) CU(cudaMemcpyAsync(out, d_out, (size_t)b.bytes, cudaMemcpyDeviceToHost, st));
    if (!on_device || !out_on_device) CU(cudaStreamSynchronize(st));
    return 0;
}

int b200pose_infer_frames(b200pose_net* net, b200pose_post* post, const b200pose_frame* frames, int n, int format,
                          int on_device, int rotate, int dest_size, int factor, const double* scales, int n_scales,
                          int mode, float thresh, int flip, void* cuda_stream) {
    if (int rc = check_infer(net, post, mode)) return rc;
    FrameBatch b;
    if (int rc = check_frames(frames, n, post->pb.batch_cap, format, rotate, &b)) return rc;
    if (flip && 2 * n > kMaxRagged) return fail("frames: %d frames with flip (2n <= %d)", n, kMaxRagged);
    const bool uniform = b.uniform();
    const int h = uniform ? b.hw[0] : 0, w = uniform ? b.hw[1] : 0;
    const int* hw = uniform ? nullptr : b.hw.data();
    if (frames_are_packed_bgr(b))
        return infer_raw(net, post, b.tab[0].plane[0], on_device, n, h, w, hw, dest_size, factor, scales, n_scales, mode,
                         thresh, flip, cuda_stream);
    return infer_raw(net, post, nullptr, on_device, n, h, w, hw, dest_size, factor, scales, n_scales, mode, thresh, flip,
                     cuda_stream, &b);
}

int b200pose_jpeg_info(const unsigned char* data, long long size, int* h, int* w, int* supported) {
    return b200pose_jpeg_info_ex(data, size, 0, h, w, supported);
}

int b200pose_jpeg_info_ex(const unsigned char* data, long long size, int progressive, int* h, int* w, int* supported) {
    if (!data || !h || !w || !supported) return fail("jpeg_info: null pointer");
    std::unique_ptr<JpegParsed> P(new JpegParsed);
    const bool ok = jpeg_parse(data, size, kJpegMaxPixels, P.get(), progressive != 0);
    *h = P->im.oh;
    *w = P->im.ow;
    *supported = ok && P->supported;
    if (!ok) return fail("jpeg: %s", P->reason);
    if (!P->supported) fail("jpeg: %s", P->reason);
    return 0;
}

int b200pose_net_decode_jpegs(b200pose_net* net, const unsigned char* const* data, const long long* sizes, int n,
                              unsigned char* out, int out_on_device, void* cuda_stream) {
    if (!net) return fail("null net");
    if (!out) return fail("decode_jpegs: null output");
    JpegCall j;
    if (int rc = check_jpegs(data, sizes, n, kMaxRagged, &j, net->jpeg_progressive)) return rc;
    CU(cudaSetDevice(net->device));
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    unsigned char* d_out = out;
    if (!out_on_device) {
        CU(net->raw_stage.ensure((size_t)j.bytes));
        d_out = net->raw_stage.p;
    }
    const unsigned* d_status;
    if (int rc = decode_jpegs_dev(net, j, d_out, st, &d_status)) return rc;
    if (!out_on_device) CU(cudaMemcpyAsync(out, d_out, (size_t)j.bytes, cudaMemcpyDeviceToHost, st));
    std::vector<unsigned> status(n);
    CU(cudaMemcpyAsync(status.data(), d_status, n * sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    for (int i = 0; i < n; ++i)
        if (status[i]) return fail("jpeg image %d: damaged entropy-coded data: %s (status %u)", i, jpeg_status_name(status[i]), status[i]);
    return 0;
}

int b200pose_infer_jpegs(b200pose_net* net, b200pose_post* post, const unsigned char* const* data,
                         const long long* sizes, int n, int dest_size, int factor, const double* scales, int n_scales,
                         int mode, float thresh, int flip, void* cuda_stream) {
    if (int rc = check_infer(net, post, mode)) return rc;
    if (flip && 2 * n > kMaxRagged) return fail("jpegs: %d images with flip (2n <= %d)", n, kMaxRagged);
    JpegCall j;
    if (int rc = check_jpegs(data, sizes, n, post->pb.batch_cap, &j, net->jpeg_progressive)) return rc;
    const bool uniform = j.uniform();
    return infer_raw(net, post, nullptr, 0, n, uniform ? j.hw[0] : 0, uniform ? j.hw[1] : 0, uniform ? nullptr : j.hw.data(),
                     dest_size, factor, scales, n_scales, mode, thresh, flip, cuda_stream, nullptr, &j);
}

int b200pose_png_info(const unsigned char* data, long long size, int* h, int* w, int* supported) {
    if (!data || !h || !w || !supported) return fail("png_info: null pointer");
    std::unique_ptr<PngParsed> P(new PngParsed);
    const bool ok = png_parse(data, size, kJpegMaxPixels, P.get());
    *h = P->im.oh;
    *w = P->im.ow;
    *supported = ok && P->supported;
    if (!ok) return fail("png: %s", P->reason);
    if (!P->supported) fail("png: %s", P->reason);
    return 0;
}

int b200pose_net_decode_pngs(b200pose_net* net, const unsigned char* const* data, const long long* sizes, int n,
                             unsigned char* out, int out_on_device, void* cuda_stream) {
    if (!net) return fail("null net");
    if (!out) return fail("decode_pngs: null output");
    PngCall j;
    if (int rc = check_pngs(data, sizes, n, kMaxRagged, &j)) return rc;
    CU(cudaSetDevice(net->device));
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    unsigned char* d_out = out;
    if (!out_on_device) {
        CU(net->raw_stage.ensure((size_t)j.bytes));
        d_out = net->raw_stage.p;
    }
    const unsigned* d_status;
    if (int rc = decode_pngs_dev(net, j, d_out, st, &d_status)) return rc;
    if (!out_on_device) CU(cudaMemcpyAsync(out, d_out, (size_t)j.bytes, cudaMemcpyDeviceToHost, st));
    std::vector<unsigned> status(n);
    CU(cudaMemcpyAsync(status.data(), d_status, n * sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    for (int i = 0; i < n; ++i)
        if (status[i]) return fail("png image %d: damaged image data: %s (status %u)", i, png_status_name(status[i]), status[i]);
    return 0;
}

int b200pose_infer_pngs(b200pose_net* net, b200pose_post* post, const unsigned char* const* data,
                        const long long* sizes, int n, int dest_size, int factor, const double* scales, int n_scales,
                        int mode, float thresh, int flip, void* cuda_stream) {
    if (int rc = check_infer(net, post, mode)) return rc;
    if (flip && 2 * n > kMaxRagged) return fail("pngs: %d images with flip (2n <= %d)", n, kMaxRagged);
    PngCall j;
    if (int rc = check_pngs(data, sizes, n, post->pb.batch_cap, &j)) return rc;
    const bool uniform = j.uniform();
    return infer_raw(net, post, nullptr, 0, n, uniform ? j.hw[0] : 0, uniform ? j.hw[1] : 0, uniform ? nullptr : j.hw.data(),
                     dest_size, factor, scales, n_scales, mode, thresh, flip, cuda_stream, nullptr, nullptr, &j);
}

// ------------------------------------------------------------------------------------------------ JPEG encoding
static int jenc_size_ok(int h, int w) { return h >= 1 && h <= 65535 && w >= 1 && w <= 65535; }

long long b200pose_jpeg_encode_bound(int h, int w, int sampling) {
    if (!jenc_size_ok(h, w)) return fail("jpeg_encode_bound: size %d x %d (1 .. 65535 each)", h, w), -1;
    if (!jenc_sampling_ok(sampling)) return fail("jpeg_encode_bound: unknown sampling 0x%X", sampling), -1;
    std::unique_ptr<JencImage> im(new JencImage);
    jenc_image(h, w, 95, sampling, im.get());
    return jenc_stream_bound(*im);
}

int b200pose_net_encode_jpegs(b200pose_net* net, const unsigned char* frames, int frames_on_device, const int* frame_hw,
                              int n, int quality, int sampling, unsigned char* out, long long out_cap, int out_on_device,
                              long long* sizes, void* cuda_stream) {
    if (!net) return fail("null net");
    if (!frames || !frame_hw || !out || !sizes) return fail("encode_jpegs: null pointer");
    if (n < 1 || n > kMaxRagged) return fail("encode_jpegs: n = %d images (1 .. %d)", n, kMaxRagged);
    if (quality < 1 || quality > 100) return fail("encode_jpegs: quality %d (1 .. 100)", quality);
    if (!jenc_sampling_ok(sampling))
        return fail("encode_jpegs: unknown sampling 0x%X (0x221111, 0x211111, 0x121111, 0x411111 or 0x111111)", sampling);
    // descriptors (header and tables built once per size of the call), then the Huffman tables, and room for the
    // per-image bit counts, stream sizes and bit-buffer offsets
    std::vector<JencImage> ims(n);
    std::map<std::pair<int, int>, int> first;
    long long src = 0, blocks = 0, bound = 0, max_blocks = 0;
    for (int i = 0; i < n; ++i) {
        const int h = frame_hw[2 * i], w = frame_hw[2 * i + 1];
        if (!jenc_size_ok(h, w)) return fail("encode_jpegs: image %d size %d x %d (1 .. 65535 each)", i, h, w);
        const auto seen = first.emplace(std::make_pair(h, w), i);
        if (seen.second) jenc_image(h, w, quality, sampling, &ims[i]);
        else ims[i] = ims[seen.first->second];
        ims[i].src = src;
        ims[i].blk0 = blocks;
        src += 3LL * h * w;
        blocks += ims[i].blocks;
        bound += jenc_stream_bound(ims[i]);
        max_blocks = std::max(max_blocks, ims[i].blocks);
    }
    if (out_cap < bound)
        return fail("encode_jpegs: out_cap %lld bytes, below %lld (b200pose_jpeg_encode_bound summed over the images)",
                    out_cap, bound);
    const size_t o_huff = n * sizeof(JencImage), o_bits = o_huff + 4 * sizeof(JencHuff);
    const size_t o_sizes = o_bits + n * sizeof(long long), o_wbase = o_sizes + n * sizeof(long long);
    std::vector<char> up(o_wbase + n * sizeof(long long));
    memcpy(up.data(), ims.data(), o_huff);
    for (int t = 0; t < 4; ++t) jenc_huff_table(t, reinterpret_cast<JencHuff*>(up.data() + o_huff) + t);
    CU(cudaSetDevice(net->device));
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    CU(net->jenc_in.ensure(up.size()));
    CU(net->jenc_coef.ensure((size_t)blocks * 64));
    CU(net->jenc_acbits.ensure((size_t)blocks));
    CU(net->jenc_off.ensure((size_t)blocks));
    if (!frames_on_device) CU(net->jenc_frames.ensure((size_t)src));
    CU(cudaMemcpyAsync(net->jenc_in.p, up.data(), up.size(), cudaMemcpyHostToDevice, st));
    if (!frames_on_device) CU(cudaMemcpyAsync(net->jenc_frames.p, frames, (size_t)src, cudaMemcpyHostToDevice, st));
    char* d = net->jenc_in.p;
    JencBatch b;
    b.ims = reinterpret_cast<const JencImage*>(d);
    b.n = n;
    b.huff = reinterpret_cast<const JencHuff*>(d + o_huff);
    b.frames = frames_on_device ? frames : net->jenc_frames.p;
    b.coef = net->jenc_coef.p;
    b.acbits = net->jenc_acbits.p;
    b.off = net->jenc_off.p;
    b.wbase = reinterpret_cast<const long long*>(d + o_wbase);
    b.words = nullptr;
    b.bits = reinterpret_cast<long long*>(d + o_bits);
    b.sizes = reinterpret_cast<long long*>(d + o_sizes);
    b.out = nullptr;
    b.max_blocks = max_blocks;
    // phase 0, then the bit buffers sized from the bit counts
    if (int rc = launched(jpeg_encode_launch(b, 0, st), "jpeg_encode_launch", 2)) return rc;
    std::vector<long long> got(n), wbase(n);
    CU(cudaMemcpyAsync(got.data(), b.bits, n * sizeof(long long), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    long long words = 0;
    for (int i = 0; i < n; ++i) {
        wbase[i] = words;
        words += jenc_words(got[i]);
    }
    CU(net->jenc_words.ensure((size_t)words));
    b.words = net->jenc_words.p;
    CU(cudaMemsetAsync(b.words, 0, (size_t)words * sizeof(unsigned), st));
    CU(cudaMemcpyAsync(d + o_wbase, wbase.data(), n * sizeof(long long), cudaMemcpyHostToDevice, st));
    // phase 1, then the output sized from the stream sizes
    if (int rc = launched(jpeg_encode_launch(b, 1, st), "jpeg_encode_launch", 2)) return rc;
    CU(cudaMemcpyAsync(got.data(), b.sizes, n * sizeof(long long), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    long long total = 0;
    for (int i = 0; i < n; ++i) total += got[i];
    if (!out_on_device) CU(net->jenc_out.ensure((size_t)total));
    b.out = out_on_device ? out : net->jenc_out.p;
    if (int rc = launched(jpeg_encode_launch(b, 2, st), "jpeg_encode_launch", 1)) return rc;
    if (!out_on_device) CU(cudaMemcpyAsync(out, net->jenc_out.p, (size_t)total, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    memcpy(sizes, got.data(), n * sizeof(long long));
    return 0;
}

// ------------------------------------------------------------------------------------------------ PNG encoding
long long b200pose_png_encode_bound(int h, int w) {
    if (!jenc_size_ok(h, w)) return fail("png_encode_bound: size %d x %d (1 .. 65535 each)", h, w), -1;
    return png_stream_bound(h, w);
}

int b200pose_net_encode_pngs(b200pose_net* net, const unsigned char* frames, int frames_on_device, const int* frame_hw,
                             int n, unsigned char* out, long long out_cap, int out_on_device, long long* sizes,
                             void* cuda_stream) {
    if (!net) return fail("null net");
    if (!frames || !frame_hw || !out || !sizes) return fail("encode_pngs: null pointer");
    if (n < 1 || n > kMaxRagged) return fail("encode_pngs: n = %d images (1 .. %d)", n, kMaxRagged);
    // descriptors, then the per-image results (zeroed) and room for the deflate word offsets
    std::vector<PngImage> ims(n);
    long long src = 0, filt = 0, tiles = 0, blocks = 0, bound = 0, max_tiles = 0, max_blocks = 0;
    for (int i = 0; i < n; ++i) {
        const int h = frame_hw[2 * i], w = frame_hw[2 * i + 1];
        if (!jenc_size_ok(h, w)) return fail("encode_pngs: image %d size %d x %d (1 .. 65535 each)", i, h, w);
        PngImage& im = ims[i];
        im.h = h;
        im.w = w;
        im.n = (long long)h * (3LL * w + 1);
        im.src = src;
        im.f0 = filt;
        im.tile0 = tiles;
        im.blk0 = blocks;
        im.tiles = (int)((im.n + kPngTile - 1) / kPngTile);
        im.max_blocks = (int)png_blocks(im.n);
        png_zlib_header(im.n, im.zhdr);
        src += 3LL * h * w;
        filt += (im.n + 15) & ~15LL;
        tiles += im.tiles;
        blocks += im.max_blocks;
        bound += png_stream_bound(h, w);
        max_tiles = std::max(max_tiles, (long long)im.tiles);
        max_blocks = std::max(max_blocks, (long long)im.max_blocks);
    }
    if (out_cap < bound)
        return fail("encode_pngs: out_cap %lld bytes, below %lld (b200pose_png_encode_bound summed over the images)",
                    out_cap, bound);
    const size_t o_outs = n * sizeof(PngImage), o_wbase = o_outs + n * sizeof(PngImageOut);
    std::vector<char> up(o_wbase + n * sizeof(long long), 0);
    memcpy(up.data(), ims.data(), o_outs);
    CU(cudaSetDevice(net->device));
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    CU(net->penc_in.ensure(up.size()));
    CU(net->penc_filt.ensure((size_t)filt));
    CU(net->penc_sym.ensure((size_t)filt));
    CU(net->penc_tiles.ensure((size_t)tiles * 6));
    CU(net->penc_blocks.ensure((size_t)blocks));
    if (!frames_on_device) CU(net->penc_frames.ensure((size_t)src));
    CU(cudaMemcpyAsync(net->penc_in.p, up.data(), up.size(), cudaMemcpyHostToDevice, st));
    if (!frames_on_device) CU(cudaMemcpyAsync(net->penc_frames.p, frames, (size_t)src, cudaMemcpyHostToDevice, st));
    char* d = net->penc_in.p;
    long long* t = net->penc_tiles.p;
    PngBatch b;
    b.ims = reinterpret_cast<const PngImage*>(d);
    b.n = n;
    b.frames = frames_on_device ? frames : net->penc_frames.p;
    b.filt = net->penc_filt.p;
    b.tfirst = t;
    b.tlast = t + tiles;
    b.tstart = t + 2 * tiles;
    b.tend = t + 3 * tiles;
    b.tcount = t + 4 * tiles;
    b.tbase = t + 5 * tiles;
    b.sym = net->penc_sym.p;
    b.blocks = net->penc_blocks.p;
    b.outs = reinterpret_cast<PngImageOut*>(d + o_outs);
    b.wbase = reinterpret_cast<const long long*>(d + o_wbase);
    b.words = nullptr;
    b.out = nullptr;
    b.max_tiles = max_tiles;
    b.max_blocks = max_blocks;
    b.max_chunks = 0;
    // phase 0, then the deflate words and the output sized from what it found
    if (int rc = launched(png_encode_launch(b, 0, st), "png_encode_launch", 7)) return rc;
    std::vector<PngImageOut> got(n);
    CU(cudaMemcpyAsync(got.data(), b.outs, n * sizeof(PngImageOut), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    std::vector<long long> wbase(n);
    long long words = 0, total = 0;
    for (int i = 0; i < n; ++i) {
        wbase[i] = words;
        words += got[i].bits / 32 + 2;
        total += got[i].size;
        b.max_chunks = std::max(b.max_chunks, (long long)got[i].chunks);
    }
    CU(net->penc_words.ensure((size_t)words));
    b.words = net->penc_words.p;
    CU(cudaMemsetAsync(b.words, 0, (size_t)words * sizeof(unsigned), st));
    CU(cudaMemcpyAsync(d + o_wbase, wbase.data(), n * sizeof(long long), cudaMemcpyHostToDevice, st));
    if (!out_on_device) CU(net->penc_out.ensure((size_t)total));
    b.out = out_on_device ? out : net->penc_out.p;
    if (int rc = launched(png_encode_launch(b, 1, st), "png_encode_launch", 2)) return rc;
    if (!out_on_device) CU(cudaMemcpyAsync(out, net->penc_out.p, (size_t)total, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    for (int i = 0; i < n; ++i) sizes[i] = got[i].size;
    return 0;
}

// ------------------------------------------------------------------------------------------------ COCO keypoint evaluation
int b200pose_coco_kpt_eval(int device, int n_units, int n_cats, const int* unit_cat, const int* unit_gt0,
                           const int* unit_dt0, const long long* gt_id, const double* gt_kpt, int gt_kpt_len,
                           const double* gt_box, const unsigned char* gt_crowd, const unsigned char* gt_ignore,
                           const double* dt_kpt, int dt_kpt_len, const double* dt_score, const double* thr,
                           double* precision, double* recall, double* oks, long long oks_cap, long long* oks_count) {
    if (n_units < 0) return fail("coco_kpt_eval: n_units = %d", n_units);
    if (n_cats < 1 || n_cats > kCocoMaxCats) return fail("coco_kpt_eval: n_cats = %d (1 .. %d)", n_cats, kCocoMaxCats);
    if ((n_units && (!unit_cat || !unit_gt0 || !unit_dt0)) || !thr || !precision || !recall)
        return fail("coco_kpt_eval: null pointer");
    if (gt_kpt_len != kCocoKpt) return fail("coco_kpt_eval: gt_kpt_len = %d (keypoints are 51 values)", gt_kpt_len);
    if (dt_kpt_len != kCocoKpt) return fail("coco_kpt_eval: dt_kpt_len = %d (keypoints are 51 values)", dt_kpt_len);
    for (int i = 0; i < kCocoIouThrs + kCocoRecThrs; ++i) {
        if (!std::isfinite(thr[i])) return fail("coco_kpt_eval: thr[%d] is not finite", i);
        if (i != 0 && i != kCocoIouThrs && thr[i] < thr[i - 1]) return fail("coco_kpt_eval: thr[%d] not ascending", i);
    }
    const int G = n_units ? unit_gt0[n_units] : 0, D = n_units ? unit_dt0[n_units] : 0;
    if (n_units && (unit_gt0[0] != 0 || unit_dt0[0] != 0)) return fail("coco_kpt_eval: unit_gt0[0] / unit_dt0[0] not 0");
    if (G > kCocoMaxTotal) return fail("coco_kpt_eval: %d gts (at most %d)", G, kCocoMaxTotal);
    if (D > kCocoMaxTotal) return fail("coco_kpt_eval: %d detections (at most %d)", D, kCocoMaxTotal);
    if ((G && (!gt_id || !gt_kpt || !gt_box || !gt_crowd || !gt_ignore)) || (D && (!dt_kpt || !dt_score)))
        return fail("coco_kpt_eval: null pointer");
    // units, kept detections and OKS blocks
    std::vector<CocoUnit> units(n_units);
    std::vector<int> cat_k0(n_cats + 1, 0);
    int kept = 0;
    long long oks_n = 0;
    for (int u = 0; u < n_units; ++u) {
        CocoUnit& x = units[u];
        x.cat = unit_cat[u];
        if (x.cat < 0 || x.cat >= n_cats) return fail("coco_kpt_eval: unit_cat[%d] = %d (0 .. %d)", u, x.cat, n_cats - 1);
        if (u && x.cat < units[u - 1].cat) return fail("coco_kpt_eval: unit_cat[%d] below the unit before", u);
        x.g0 = unit_gt0[u];
        x.ng = unit_gt0[u + 1] - x.g0;
        x.d0 = unit_dt0[u];
        x.nd = unit_dt0[u + 1] - x.d0;
        if (x.ng < 0 || x.ng > kCocoMaxUnitGts) return fail("coco_kpt_eval: unit_gt0: unit %d has %d gts (0 .. %d)", u, x.ng, kCocoMaxUnitGts);
        if (x.nd < 0 || x.nd > kCocoMaxUnitDets)
            return fail("coco_kpt_eval: unit_dt0: unit %d has %d detections (0 .. %d)", u, x.nd, kCocoMaxUnitDets);
        x.nk = std::min(x.nd, kCocoMaxDets);
        x.k0 = kept;
        x.o0 = oks_n;
        kept += x.nk;
        oks_n += (long long)x.nk * x.ng;
        if (kept > kCocoMaxKept) return fail("coco_kpt_eval: more than %d detections after the cut to 20 per unit", kCocoMaxKept);
        cat_k0[x.cat + 1] = kept;
    }
    for (int c = 1; c <= n_cats; ++c) cat_k0[c] = std::max(cat_k0[c], cat_k0[c - 1]);
    if (oks && oks_cap < oks_n) return fail("coco_kpt_eval: oks_cap %lld doubles, below %lld", oks_cap, oks_n);
    std::set<long long> ids;
    for (int g = 0; g < G; ++g) {
        if (gt_id[g] == 0) return fail("coco_kpt_eval: gt_id[%d] is 0 (a match is marked by the gt id)", g);
        if (!ids.insert(gt_id[g]).second) return fail("coco_kpt_eval: gt_id[%d] = %lld repeats an earlier gt", g, gt_id[g]);
        for (int k = 0; k < kCocoKpt; ++k)
            if (!std::isfinite(gt_kpt[(size_t)g * kCocoKpt + k])) return fail("coco_kpt_eval: gt_kpt of gt %d is not finite", g);
        for (int k = 0; k < 5; ++k)
            if (!std::isfinite(gt_box[(size_t)g * 5 + k])) return fail("coco_kpt_eval: gt_box of gt %d is not finite", g);
    }
    for (int d = 0; d < D; ++d) {
        if (!std::isfinite(dt_score[d])) return fail("coco_kpt_eval: dt_score[%d] is not finite", d);
        for (int k = 0; k < kCocoKpt; ++k)
            if (!std::isfinite(dt_kpt[(size_t)d * kCocoKpt + k])) return fail("coco_kpt_eval: dt_kpt of detection %d is not finite", d);
    }
    // one upload: units, category offsets, gts, detections, thresholds; then the device's own arrays
    auto align = [](size_t o) { return (o + 255) & ~(size_t)255; };
    size_t at = 0;
    auto take = [&](size_t bytes) { const size_t o = at; at = align(at + bytes); return o; };
    const size_t o_units = take(n_units * sizeof(CocoUnit)), o_catk = take((n_cats + 1) * sizeof(int));
    const size_t o_gkpt = take((size_t)G * kCocoKpt * 8), o_gbox = take((size_t)G * 5 * 8), o_gflag = take(G);
    const size_t o_dkpt = take((size_t)D * kCocoKpt * 8), o_dsc = take((size_t)D * 8);
    const size_t o_thr = take((kCocoIouThrs + kCocoRecThrs) * 8), up_bytes = at;
    const size_t o_npig = take((size_t)n_cats * kCocoAreas * 4), o_kscore = take((size_t)kept * 8);
    const size_t o_karea = take((size_t)kept * 8), o_kcat = take((size_t)kept * 4), o_oks = take((size_t)oks_n * 8);
    const size_t o_state = take((size_t)kCocoAreas * kCocoIouThrs * kept), o_order = take((size_t)kept * 4);
    const size_t n_prec = (size_t)kCocoIouThrs * kCocoRecThrs * n_cats * kCocoAreas;
    const size_t n_rec = (size_t)kCocoIouThrs * n_cats * kCocoAreas;
    const size_t o_prec = take(n_prec * 8), o_rec = take(n_rec * 8);
    std::vector<char> up(up_bytes, 0);
    memcpy(up.data() + o_units, units.data(), n_units * sizeof(CocoUnit));
    memcpy(up.data() + o_catk, cat_k0.data(), (n_cats + 1) * sizeof(int));
    if (G) {
        memcpy(up.data() + o_gkpt, gt_kpt, (size_t)G * kCocoKpt * 8);
        memcpy(up.data() + o_gbox, gt_box, (size_t)G * 5 * 8);
        for (int g = 0; g < G; ++g) up[o_gflag + g] = (char)((gt_crowd[g] ? 1 : 0) | (gt_ignore[g] ? 2 : 0));
    }
    if (D) {
        memcpy(up.data() + o_dkpt, dt_kpt, (size_t)D * kCocoKpt * 8);
        memcpy(up.data() + o_dsc, dt_score, (size_t)D * 8);
    }
    memcpy(up.data() + o_thr, thr, (kCocoIouThrs + kCocoRecThrs) * 8);
    CU(cudaSetDevice(device));
    Stream st;
    CU(cudaStreamCreateWithFlags(&st.h, cudaStreamNonBlocking));
    DevBuf<char> buf;
    CU(buf.ensure(at));
    char* d = buf.p;
    CU(cudaMemcpyAsync(d, up.data(), up_bytes, cudaMemcpyHostToDevice, st));
    CU(cudaMemsetAsync(d + o_npig, 0, (size_t)n_cats * kCocoAreas * 4, st));
    CocoBatch b;
    b.units = reinterpret_cast<const CocoUnit*>(d + o_units);
    b.n_units = n_units;
    b.n_cats = n_cats;
    b.cat_k0 = reinterpret_cast<const int*>(d + o_catk);
    b.gt_kpt = reinterpret_cast<const double*>(d + o_gkpt);
    b.gt_box = reinterpret_cast<const double*>(d + o_gbox);
    b.gt_flag = reinterpret_cast<const unsigned char*>(d + o_gflag);
    b.dt_kpt = reinterpret_cast<const double*>(d + o_dkpt);
    b.dt_score = reinterpret_cast<const double*>(d + o_dsc);
    b.thr = reinterpret_cast<const double*>(d + o_thr);
    b.kept = kept;
    b.k_score = reinterpret_cast<double*>(d + o_kscore);
    b.k_area = reinterpret_cast<double*>(d + o_karea);
    b.k_cat = reinterpret_cast<int*>(d + o_kcat);
    b.oks = reinterpret_cast<double*>(d + o_oks);
    b.state = reinterpret_cast<unsigned char*>(d + o_state);
    b.order = reinterpret_cast<int*>(d + o_order);
    b.npig = reinterpret_cast<int*>(d + o_npig);
    b.precision = reinterpret_cast<double*>(d + o_prec);
    b.recall = reinterpret_cast<double*>(d + o_rec);
    if (int rc = launched(coco_eval_launch(b, st), "coco_eval_launch", kCocoLaunches)) return rc;
    CU(cudaMemcpyAsync(precision, b.precision, n_prec * 8, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(recall, b.recall, n_rec * 8, cudaMemcpyDeviceToHost, st));
    if (oks && oks_n) CU(cudaMemcpyAsync(oks, b.oks, (size_t)oks_n * 8, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    if (oks_count) *oks_count = oks_n;
    return 0;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------ training targets, stage losses
namespace {
// b200pose_ground_truth with keypoints of type T (float32, or float64 after a flip)
template <class T>
int ground_truth_impl(int device, const T* keypoints, const int* persons, const int* hw, int n, float* heat, float* paf,
                      int canvas_h, int canvas_w, void* cuda_stream) {
    if (n < 1 || n > kGtMaxImages) return fail("ground_truth: %d images (1 .. %d)", n, kGtMaxImages);
    if (!persons || !hw) return fail("ground_truth: null persons / sizes");
    long long total = 0;
    int gh_max = 0, gw_max = 0;
    for (int i = 0; i < n; ++i) {
        if (persons[i] < 0 || persons[i] > kGtMaxPersons)
            return fail("ground_truth: persons of image %d = %d (0 .. %d)", i, persons[i], kGtMaxPersons);
        if (hw[2 * i] < kGtStride || hw[2 * i] > kGtMaxSize || hw[2 * i + 1] < kGtStride || hw[2 * i + 1] > kGtMaxSize)
            return fail("ground_truth: sizes of image %d = %d x %d (each side %d .. %d)", i, hw[2 * i], hw[2 * i + 1],
                        kGtStride, kGtMaxSize);
        total += persons[i];
        gh_max = std::max(gh_max, gt_grid(hw[2 * i]));
        gw_max = std::max(gw_max, gt_grid(hw[2 * i + 1]));
    }
    if (total && !keypoints) return fail("ground_truth: null keypoints");
    for (long long k = 0; k < total * kGtCocoParts * 3; ++k)
        if (!std::isfinite(keypoints[k]))
            return fail("ground_truth: keypoints of person %lld (of the call) are not finite", k / (kGtCocoParts * 3));
    if (canvas_h < gh_max || canvas_w < gw_max)
        return fail("ground_truth: canvas %d x %d below the largest grid %d x %d", canvas_h, canvas_w, gh_max, gw_max);
    if (canvas_h > kGtMaxSize / kGtStride || canvas_w > kGtMaxSize / kGtStride)
        return fail("ground_truth: canvas %d x %d above %d x %d cells", canvas_h, canvas_w, kGtMaxSize / kGtStride,
                    kGtMaxSize / kGtStride);
    if (!heat && !paf) return 0;      // arguments checked, nothing to write
    if (!heat || !paf) return fail("ground_truth: null heat / paf");
    // one upload: the images, then every person's 18 joints (add_neck, our_order, remove_illegal_joint on the host)
    const size_t o_joints = ((size_t)n * sizeof(GtImage) + 255) & ~(size_t)255;
    std::vector<char> up(o_joints + (size_t)total * kGtParts * 3 * sizeof(T));
    GtImage* im = reinterpret_cast<GtImage*>(up.data());
    T* jo = reinterpret_cast<T*>(up.data() + o_joints);
    for (int i = 0, j0 = 0; i < n; j0 += persons[i++]) {
        im[i] = {j0, persons[i], gt_grid(hw[2 * i]), gt_grid(hw[2 * i + 1])};
        for (int p = j0; p < j0 + persons[i]; ++p)
            gt_person_joints(keypoints + (size_t)p * kGtCocoParts * 3, hw[2 * i + 1], hw[2 * i], jo + (size_t)p * kGtParts * 3);
    }
    CU(cudaSetDevice(device));
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    void* d = nullptr;
    CU(cudaMallocAsync(&d, up.size(), st));
    GtBatch b;
    b.images = reinterpret_cast<const GtImage*>(d);
    b.joints = static_cast<char*>(d) + o_joints;
    b.f64 = sizeof(T) == 8;
    b.n = n;
    b.ch = canvas_h;
    b.cw = canvas_w;
    b.heat = heat;
    b.paf = paf;
    cudaError_t e = cudaMemcpyAsync(d, up.data(), up.size(), cudaMemcpyHostToDevice, st);
    int rc = e != cudaSuccess ? cuda_fail("ground_truth: upload: %s", cudaGetErrorString(e))
                              : launched(gt_launch(b, st), "gt_launch", kGtLaunches);
    cudaError_t ef = cudaFreeAsync(d, st);
    if (!rc && ef != cudaSuccess) rc = cuda_fail("ground_truth: cudaFreeAsync: %s", cudaGetErrorString(ef));
    return rc;
}
}  // namespace

extern "C" {
int b200pose_ground_truth(int device, const float* keypoints, const int* persons, const int* hw, int n, float* heat,
                          float* paf, int canvas_h, int canvas_w, void* cuda_stream) {
    return ground_truth_impl(device, keypoints, persons, hw, n, heat, paf, canvas_h, canvas_w, cuda_stream);
}

int b200pose_ground_truth_f64(int device, const double* keypoints, const int* persons, const int* hw, int n,
                              float* heat, float* paf, int canvas_h, int canvas_w, void* cuda_stream) {
    return ground_truth_impl(device, keypoints, persons, hw, n, heat, paf, canvas_h, canvas_w, cuda_stream);
}

// ------------------------------------------------------------------------------------------------ training batches
int b200pose_net_augment(b200pose_net* net, const unsigned char* frames, int frames_on_device, int n, const int* hw,
                         const double* params, int edge, float* out_f32, unsigned char* out_u8, int out_on_device,
                         void* cuda_stream) {
    if (!net) return fail("null net");
    if (n < 1 || n > kAugMaxImages) return fail("augment: n = %d images (1 .. %d)", n, kAugMaxImages);
    if (!frames || !hw || !params || !out_f32) return fail("augment: null frames / hw / params / out_f32");
    if (edge % 8 || edge < kAugMinEdge || edge > kAugMaxEdge)
        return fail("augment: edge %d (a multiple of 8, %d .. %d)", edge, kAugMinEdge, kAugMaxEdge);
    std::vector<AugImage> im(n);
    std::vector<int> jpeg;
    long long src_bytes = 0, tmp_bytes = 0;
    int max_tmp = 0;
    for (int i = 0; i < n; ++i) {
        const int h = hw[2 * i], w = hw[2 * i + 1];
        if (h < kAugMinSide || h > kAugMaxSide || w < kAugMinSide || w > kAugMaxSide)
            return fail("augment: size of image %d = %d x %d (each side %d .. %d)", i, h, w, kAugMinSide, kAugMaxSide);
        const double* p = params + (size_t)i * B200POSE_AUG_PARAMS;
        for (int k = 0; k < B200POSE_AUG_PARAMS; ++k)
            if (!std::isfinite(p[k]) || ((k < 9 || k > 12) && p[k] != std::floor(p[k])) || std::fabs(p[k]) > 1e6)
                return fail("augment: params[%d][%d] = %g (finite; an integer except the factors)", i, k, p[k]);
        AugImage& a = im[i];
        a.h = h;
        a.w = w;
        a.flip = (int)p[0];
        a.rw = (int)p[1];
        a.rh = (int)p[2];
        a.x0 = (int)p[3];
        a.y0 = (int)p[4];
        const int jp = (int)p[13];
        a.gray = (int)p[14];
        a.mx0 = (int)p[15];
        a.my0 = (int)p[16];
        a.mx1 = (int)p[17];
        a.my1 = (int)p[18];
        if ((a.flip | jp | a.gray) & ~1) return fail("augment: image %d: hflip, jpeg, grayscale must be 0 or 1", i);
        if (a.rw < w / 2 || a.rw > w || a.rh < h / 2 || a.rh > h || a.rw < 1 || a.rh < 1)
            return fail("augment: image %d: resized %d x %d outside %d x %d .. %d x %d", i, a.rh, a.rw, h / 2, w / 2, h, w);
        if (a.x0 < 0 || a.x0 > std::max(0, a.rw - edge) || a.y0 < 0 || a.y0 > std::max(0, a.rh - edge))
            return fail("augment: image %d: crop (%d, %d) outside the resized %d x %d image", i, a.x0, a.y0, a.rh, a.rw);
        unsigned seen = 0;
        for (int o = 0; o < 4; ++o) {
            const int op = (int)p[5 + o];
            if (op < 0 || op > 3 || (seen >> op & 1)) return fail("augment: image %d: order is not a permutation of 0 .. 3", i);
            seen |= 1u << op;
            a.order[o] = op;
        }
        for (int k = 0; k < 3; ++k) {
            if (p[9 + k] < 0) return fail("augment: image %d: factor %d = %g is negative", i, k, p[9 + k]);
            a.f[k] = p[9 + k];
        }
        a.f[3] = 0.0;
        if (p[12] < -0.5 || p[12] > 0.5) return fail("augment: image %d: hue %g outside -0.5 .. 0.5", i, p[12]);
        a.dh = (int)(p[12] * 255.0) & 255;      // np.int32(hue * 255).astype(uint8)
        if (a.mx0 < 0 || a.mx0 > a.mx1 || a.mx1 > edge || a.my0 < 0 || a.my0 > a.my1 || a.my1 > edge)
            return fail("augment: image %d: mask (%d, %d) .. (%d, %d) outside 0 .. %d", i, a.mx0, a.my0, a.mx1, a.my1, edge);
        a.cw = std::min(edge, a.rw - a.x0);
        a.ch = std::min(edge, a.rh - a.y0);
        a.left = (edge - a.cw) / 2;
        a.top = (edge - a.ch) / 2;
        int32_t k[kAugMaxTaps];
        int first, last;
        aug_taps(h, a.rh, a.y0, &first, k);
        const int cnt = aug_taps(h, a.rh, a.y0 + a.ch - 1, &last, k);
        a.r0 = first;
        a.rows = last + cnt - first;
        a.src = src_bytes;
        a.tmp = tmp_bytes;
        src_bytes += (long long)h * w * 3;
        tmp_bytes += (long long)a.rows * a.cw * 3;
        max_tmp = std::max(max_tmp, a.rows * a.cw);
        if (jp) jpeg.push_back(i);
    }
    CU(cudaSetDevice(net->device));
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    const size_t frame = (size_t)edge * edge * 3, o_sum = ((size_t)n * sizeof(AugImage) + 255) & ~(size_t)255;
    CU(net->aug_in.ensure(o_sum + (size_t)n * 8));
    AugBatch b;
    b.images = reinterpret_cast<const AugImage*>(net->aug_in.p);
    b.lsum = reinterpret_cast<unsigned long long*>(net->aug_in.p + o_sum);
    b.src = frames;
    if (!frames_on_device) {
        CU(net->aug_src.ensure((size_t)src_bytes));
        CU(cudaMemcpyAsync(net->aug_src.p, frames, (size_t)src_bytes, cudaMemcpyHostToDevice, st));
        b.src = net->aug_src.p;
    }
    CU(net->aug_tmp.ensure((size_t)tmp_bytes));
    CU(net->aug_px.ensure((size_t)n * frame));
    b.tmp = net->aug_tmp.p;
    b.px = net->aug_px.p;
    b.out = out_f32;
    b.out_u8 = out_u8;
    if (!out_on_device) {
        CU(net->aug_out.ensure((size_t)n * frame));
        b.out = net->aug_out.p;
        if (out_u8) {
            CU(net->aug_u8.ensure((size_t)n * frame));
            b.out_u8 = net->aug_u8.p;
        }
    }
    b.n = n;
    b.edge = edge;
    b.max_tmp_px = max_tmp;
    CU(cudaMemcpyAsync(net->aug_in.p, im.data(), (size_t)n * sizeof(AugImage), cudaMemcpyHostToDevice, st));
    CU(cudaMemsetAsync(b.lsum, 0, (size_t)n * 8, st));
    if (int rc = launched(aug_jitter_launch(b, st), "aug_jitter_launch", kAugLaunchesJitter)) return rc;
    if (!jpeg.empty()) {
        // jpeg_compression_augmentation: Pillow's save(quality=50) + Image.open equal cv2.imencode(q=50, 4:2:0) +
        // cv2.imdecode, which the device encoder and decoder reproduce.  The sampled images go through them packed.
        const int nj = (int)jpeg.size();
        CU(net->aug_jpeg.ensure((size_t)nj * frame));
        for (int k = 0; k < nj; ++k)
            CU(cudaMemcpyAsync(net->aug_jpeg.p + k * frame, net->aug_px.p + jpeg[k] * frame, frame,
                               cudaMemcpyDeviceToDevice, st));
        const int sampling = 0x221111;
        const long long bound = b200pose_jpeg_encode_bound(edge, edge, sampling);
        if (bound < 0) return 1;
        std::vector<unsigned char> streams((size_t)bound * nj);
        std::vector<long long> lens(nj);
        std::vector<int> jhw(2 * nj, edge);
        if (int rc = b200pose_net_encode_jpegs(net, net->aug_jpeg.p, 1, jhw.data(), nj, 50, sampling, streams.data(),
                                               bound * nj, 0, lens.data(), st))
            return rc;
        std::vector<const unsigned char*> ptrs(nj);
        for (int k = 0, at = 0; k < nj; at += (int)lens[k++]) ptrs[k] = streams.data() + at;
        if (int rc = b200pose_net_decode_jpegs(net, ptrs.data(), lens.data(), nj, net->aug_jpeg.p, 1, st)) return rc;
        for (int k = 0; k < nj; ++k)
            CU(cudaMemcpyAsync(net->aug_px.p + jpeg[k] * frame, net->aug_jpeg.p + k * frame, frame,
                               cudaMemcpyDeviceToDevice, st));
    }
    if (int rc = launched(aug_finish_launch(b, st), "aug_finish_launch", kAugLaunchesFinish)) return rc;
    if (!out_on_device) {
        CU(cudaMemcpyAsync(out_f32, b.out, (size_t)n * frame * 4, cudaMemcpyDeviceToHost, st));
        if (out_u8) CU(cudaMemcpyAsync(out_u8, b.out_u8, (size_t)n * frame, cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
    }
    return 0;
}

int b200pose_net_last_forward(b200pose_net* net, int* info, int* hw, int hw_cap) {
    if (!net || net->last.n == 0) return fail("last_forward: no forward has run");
    if (!info) return fail("last_forward: null info");
    const LastForward& l = net->last;
    info[0] = l.n;
    info[1] = l.H;
    info[2] = l.W;
    info[3] = net->arch.out[l.stages].maps;
    if (hw) {
        if (hw_cap < 2 * l.n) return fail("last_forward: hw_cap %d below 2 x %d images", hw_cap, l.n);
        for (int i = 0; i < l.n; ++i) {
            hw[2 * i] = l.ext_host.empty() ? l.H : l.ext_host[2 * i];
            hw[2 * i + 1] = l.ext_host.empty() ? l.W : l.ext_host[2 * i + 1];
        }
    }
    return 0;
}

int b200pose_net_stage_losses(b200pose_net* net, const float* heat, const float* paf, double* sums, int maps,
                              float* extrema, void* cuda_stream) {
    if (!net || net->last.n == 0) return fail("stage_losses: no forward has run");
    if (!heat || !paf) return fail("stage_losses: null heat / paf targets");
    if (!sums || !extrema) return fail("stage_losses: null sums / extrema");
    const auto& out = net->arch.out[net->last.stages];
    if (maps != out.maps)
        return fail("stage_losses: maps = %d, but the last forward wrote %d stage maps (sums is [n][%d])", maps, out.maps,
                    out.maps);
    GtLossBatch b;
    b.n_maps = out.maps;
    for (int m = 0; m < kGtMaxMaps; ++m) {
        b.maps[m] = m < out.maps ? net->out_f32[m].p : nullptr;
        b.ch[m] = m < out.maps ? net->arch.map_ch[m] : 0;
    }
    b.n = net->last.n;
    b.mh = net->last.H / 8;
    b.mw = net->last.W / 8;
    b.ext = net->last.ext;
    b.last_paf = out.paf;
    b.last_heat = out.heat;
    b.heat = heat;
    b.paf = paf;
    b.sums = sums;
    b.extrema = extrema;
    CU(cudaSetDevice(net->device));
    return launched(gt_stage_loss_launch(b, static_cast<cudaStream_t>(cuda_stream)), "gt_stage_loss_launch");
}

// ------------------------------------------------------------------------------------------------ legacy pafprocess
namespace {
std::mutex g_legacy_mu;
b200pose_post* g_legacy = nullptr;
std::vector<float> g_leg_humans;       // [nh][73]
std::vector<float> g_leg_peaks;        // by id: x, y, score
int g_leg_nh = 0;
}  // namespace

int process_paf(int p1, int p2, int p3, float* peaks, int h1, int h2, int h3, float* heatmap, int f1, int f2, int f3,
                float* pafmap) {
    (void)h2; (void)h3; (void)heatmap;
    std::lock_guard<std::mutex> lk(g_legacy_mu);
    g_leg_nh = 0;
    if (p3 != 5) return fail("process_paf: peaks must be [p1,p2,5]");
    if (f3 != 38) return fail("process_paf: pafmap must have 38 channels");
    const int P = p1 * p2;
    int dev = 0;
    cudaGetDevice(&dev);
    const int cap = 2048;
    if (!g_legacy) {
        if (b200pose_post_create(&g_legacy, dev, 1, cap, 4096)) return 2;
    }
    b200pose_post* p = g_legacy;
    CU(cudaSetDevice(p->device));
    // bucket by part (pafprocess.cpp:24-43); ids follow input order, which equals part order for the array
    // paf_to_pose_cpp builds (we require that order, the reference silently mis-indexes otherwise)
    std::vector<int> counts(18, 0), hx((size_t)18 * cap), hy((size_t)18 * cap);
    std::vector<float> hs((size_t)18 * cap);
    int prev_part = 0;
    g_leg_peaks.assign((size_t)P * 3, 0.f);
    for (int i = 0; i < P; ++i) {
        const float* r = peaks + (size_t)i * 5;
        const int part = (int)r[4];
        if (part < 0 || part >= 18) return fail("process_paf: part id %d out of range", part);
        if (part < prev_part) return fail("process_paf: peaks must be ordered by part");
        prev_part = part;
        if (counts[part] >= cap) return fail("process_paf: more than %d peaks for part %d", cap, part);
        const size_t o = (size_t)part * cap + counts[part]++;
        hx[o] = (int)r[0]; hy[o] = (int)r[1]; hs[o] = r[2];
        g_leg_peaks[3 * i] = (float)(int)r[0]; g_leg_peaks[3 * i + 1] = (float)(int)r[1]; g_leg_peaks[3 * i + 2] = r[2];
    }
    const PostBuffers& pb = p->pb;
    cudaStream_t st = nullptr;
    if (p->runs > 0) CU(cudaStreamWaitEvent(st, p->ev_fetch[(p->runs - 1) & 1], 0));   // previous call's second-stream work
    CU(cudaMemsetAsync(pb.status, 0, sizeof(int), st));
    CU(cudaMemcpyAsync(pb.counts, counts.data(), 18 * sizeof(int), cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(pb.peak_x, hx.data(), hx.size() * 4, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(pb.peak_y, hy.data(), hy.size() * 4, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(pb.peak_s, hs.data(), hs.size() * 4, cudaMemcpyHostToDevice, st));
    CU(p->d_paf.ensure((size_t)f1 * f2 * f3));
    CU(cudaMemcpyAsync(p->d_paf.p, pafmap, (size_t)f1 * f2 * f3 * 4, cudaMemcpyHostToDevice, st));
    // the reference's drop-in keeps the reference's constants (g_legacy's settings are never changed either)
    if (launched(post_limbs(pb, 1, p->d_paf.p, 0, 1, (long)f2 * f3, f3, 0, h1, f2, f1, st), "post_limbs")) return 1;
    if (enqueue_assemble_and_fetch(p, 1, st, nullptr)) return 3;
    if (b200pose_post_sync(p)) return 3;
    const int status = p->hp_status[p->cur].p[0];
    if (status & 0xff & ~16) return fail("process_paf: capacity exceeded (status %d)", status);
    g_leg_nh = p->hp_nh[p->cur].p[0];
    const float* humans = p->hp_humans[p->cur].p;
    g_leg_humans.assign(humans, humans + (size_t)g_leg_nh * kHumanFloats);
    return 0;
}
// The reference's getters index its vectors unchecked (pafprocess.cpp:196-218); out-of-range arguments return -1 / 0 here.
static bool leg_human_ok(int human_id) { return human_id >= 0 && human_id < g_leg_nh; }
static bool leg_cid_ok(int cid) { return cid >= 0 && (size_t)cid * 3 + 2 < g_leg_peaks.size(); }
int get_num_humans(void) { return g_leg_nh; }
int get_part_cid(int human_id, int part_id) {
    if (!leg_human_ok(human_id) || part_id < 0 || part_id >= 18) return -1;
    return (int)g_leg_humans[(size_t)human_id * kHumanFloats + 1 + 4 * part_id + 3];
}
float get_score(int human_id) { return leg_human_ok(human_id) ? g_leg_humans[(size_t)human_id * kHumanFloats] : 0.f; }
int get_part_x(int cid) { return leg_cid_ok(cid) ? (int)g_leg_peaks[3 * (size_t)cid] : -1; }
int get_part_y(int cid) { return leg_cid_ok(cid) ? (int)g_leg_peaks[3 * (size_t)cid + 1] : -1; }
float get_part_score(int cid) { return leg_cid_ok(cid) ? g_leg_peaks[3 * (size_t)cid + 2] : 0.f; }

}  // extern "C"
