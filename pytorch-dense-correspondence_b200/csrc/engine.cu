// Network-level orchestration of the dilated backbones' forward/backward behind the C ABI, plus the single-operator
// entry points.  The structure restated here is the reference's
//   PSD/vision/torchvision/models/resnet.py:112-265  (ResNet.__init__/_make_layer/forward, BasicBlock :53-69, Bottleneck :72-109)
//   PSD/pytorch_segmentation_detection/models/resnet_dilated.py:283-322 (Resnet34_8s), :399-435 (Resnet50_8s)
// configured as resnet34 / resnet50(fully_conv=True, output_stride=8, remove_avg_pool_layer=True).
#include <algorithm>
#include <cstring>
#include <deque>
#include <mutex>
#include <string>
#include <vector>

#include "conv.cuh"
#include "conv_tc.cuh"

namespace ddn {

std::atomic<long long> g_launches{0};
static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

// SMs left free by the persistent tensor-core kernels (one CTA per SM, no room for a second): while a data-parallel host has a gradient
// all-reduce in flight, NCCL's CTAs need somewhere to run -- without the reservation they take SMs between two of our launches and
// the next persistent kernel runs a whole extra wave for the CTAs that found no SM.  Set by ddn_set_reserved_sms (DDN_RESERVED_SMS).
static std::atomic<int> g_reserved_sms{-1};
// ... and the same for a WINDOW only: from the first gradient bucket a backward hands to its host (whose all-reduce then runs
// concurrently) to the end of that backward (DDN_OVERLAP_RESERVED_SMS = n; the host then caps NCCL at n CTAs).  Default 0
// (no reservation, NCCL's own CTA count); the effect has not been measured on H100.
static std::atomic<int> g_window_reserved{0};
static int overlap_window_sms() {
  static int v = -1;
  if (v < 0) { const char* e = getenv("DDN_OVERLAP_RESERVED_SMS"); v = e ? atoi(e) : 0; if (v < 0 || v > 64) v = 0; }
  return v;
}
int tc_worker_sms() {
  int r = g_reserved_sms.load(std::memory_order_relaxed);
  if (r < 0) { const char* e = getenv("DDN_RESERVED_SMS"); r = e ? atoi(e) : 0; if (r < 0) r = 0; g_reserved_sms.store(r); }
  r = std::max(r, g_window_reserved.load(std::memory_order_relaxed));
  const int n = num_sms();
  return r >= n - 8 ? 8 : n - r;
}

int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
      n = 132;                 // H100 SXM
  }
  return n;
}

// ------------------------------------------------------------------------------------------------ profiler
static const char* kProfNames[PROF_NUM_CLASSES] = {"conv_fwd_simt", "conv_dgrad_simt", "conv_wgrad_simt", "conv_fwd_tc",
                                                   "conv_dgrad_tc", "conv_wgrad_tc", "loss_fwd", "loss_bwd"};
struct ProfRec { int cls; double work; cudaEvent_t a, b; };
static std::mutex g_prof_mu;
static std::vector<ProfRec> g_prof;
static size_t g_prof_used = 0;
static std::atomic<int> g_prof_on{0};

ProfScope::ProfScope(int cls, double work, cudaStream_t s) : slot(-1), st(s) {
  if (!g_prof_on.load(std::memory_order_relaxed)) return;
  std::lock_guard<std::mutex> lk(g_prof_mu);
  if (g_prof_used == g_prof.size()) {
    if (g_prof.size() >= (1u << 17)) return;
    ProfRec r; r.cls = cls; r.work = work;
    if (cudaEventCreate(&r.a) != cudaSuccess || cudaEventCreate(&r.b) != cudaSuccess) return;
    g_prof.push_back(r);
  }
  slot = (int)g_prof_used++;
  g_prof[slot].cls = cls; g_prof[slot].work = work;
  cudaEventRecord(g_prof[slot].a, st);
}
ProfScope::~ProfScope() {
  if (slot < 0) return;
  std::lock_guard<std::mutex> lk(g_prof_mu);
  cudaEventRecord(g_prof[slot].b, st);
}

// ------------------------------------------------------------------------------------------------ network description
struct ConvSpec { int cin, cout, k, stride, pad, dil; int64_t w_off; };
struct BnSpec { int C; int64_t g_off, b_off, rm_off, rv_off; };
// main branch: c[0..n) each followed by b[0..n) (ReLU after all but the last, which takes the residual first);
// BasicBlock: n = 2 (3x3, 3x3), Bottleneck: n = 3 (1x1, 3x3 carrying the stride and dilation, 1x1 expanding to 4 x planes)
struct BlockSpec { int n; ConvSpec c[3], ds; BnSpec b[3], bd; bool has_ds; };

struct NetSpec {
  int arch = 0, D = 0;
  ConvSpec stem; BnSpec stem_bn;
  std::vector<BlockSpec> blocks;
  int layer_first[4] = {0, 0, 0, 0};    // index of each residual layer's first block
  int max_c = 0;                        // widest BatchNorm (sizes the statistics accumulator and the column-sum slots)
  int fc_cin = 0;                       // channels of the trunk output (the fc input)
  int64_t fc_w = 0, fc_b = 0, n_params = 0, n_buffers = 0;
  std::vector<ddn_tensor_entry> ptab, btab;
};

static void add_entry(std::vector<ddn_tensor_entry>& tab, int64_t& cursor, const std::string& name,
                      std::initializer_list<int> shape, int64_t* off_out) {
  ddn_tensor_entry e;
  memset(&e, 0, sizeof(e));
  snprintf(e.name, sizeof(e.name), "%s", name.c_str());
  e.ndim = (int)shape.size();
  int64_t n = 1; int i = 0;
  for (int s : shape) { e.shape[i++] = s; n *= s; }
  e.offset = cursor; e.numel = n;
  *off_out = cursor;
  cursor += (n + 3) / 4 * 4;   // keep every tensor 16-byte aligned inside the flat array
  tab.push_back(e);
}

static NetSpec build_spec(int arch, int D) {
  NetSpec s; s.arch = arch; s.D = D;
  const bool bottleneck = arch == DDN_ARCH_RESNET50_8S;
  const int expansion = bottleneck ? 4 : 1;
  int64_t pc = 0, bc = 0;
  auto conv = [&](const std::string& name, int cin, int cout, int k, int stride, int pad, int dil) {
    ConvSpec c{cin, cout, k, stride, pad, dil, 0};
    add_entry(s.ptab, pc, name + ".weight", {cout, cin, k, k}, &c.w_off);
    return c;
  };
  auto bn = [&](const std::string& name, int C) {
    BnSpec b{C, 0, 0, 0, 0};
    add_entry(s.ptab, pc, name + ".weight", {C}, &b.g_off);
    add_entry(s.ptab, pc, name + ".bias", {C}, &b.b_off);
    add_entry(s.btab, bc, name + ".running_mean", {C}, &b.rm_off);
    add_entry(s.btab, bc, name + ".running_var", {C}, &b.rv_off);
    return b;
  };
  s.stem = conv("conv1", 3, 64, 7, 2, 3, 1);
  s.stem_bn = bn("bn1", 64);
  // resnet.py:183-229 with output_stride = 8
  const int layers[4] = {3, 4, 6, 3}, planes[4] = {64, 128, 256, 512}, strides[4] = {1, 2, 2, 2};
  int inplanes = 64, current_stride = 4, current_dilation = 1;
  for (int L = 0; L < 4; ++L) {
    int stride = strides[L];
    const int out_c = planes[L] * expansion;
    bool ds = stride != 1 || inplanes != out_c;
    if (ds) {
      if (current_stride == 8) { current_dilation *= stride; stride = 1; }
      else current_stride *= stride;
    }
    s.layer_first[L] = (int)s.blocks.size();
    for (int i = 0; i < layers[L]; ++i) {
      std::string p = "layer" + std::to_string(L + 1) + "." + std::to_string(i);
      BlockSpec b; memset(&b, 0, sizeof(b));
      int st = i == 0 ? stride : 1;
      int dil = current_dilation;
      if (bottleneck) {       // resnet.py:72-109: the stride sits on conv2, the 3x3
        b.n = 3;
        b.c[0] = conv(p + ".conv1", inplanes, planes[L], 1, 1, 0, 1);
        b.b[0] = bn(p + ".bn1", planes[L]);
        b.c[1] = conv(p + ".conv2", planes[L], planes[L], 3, st, dil, dil);
        b.b[1] = bn(p + ".bn2", planes[L]);
        b.c[2] = conv(p + ".conv3", planes[L], out_c, 1, 1, 0, 1);
        b.b[2] = bn(p + ".bn3", out_c);
      } else {
        b.n = 2;
        b.c[0] = conv(p + ".conv1", inplanes, planes[L], 3, st, dil, dil);
        b.b[0] = bn(p + ".bn1", planes[L]);
        b.c[1] = conv(p + ".conv2", planes[L], planes[L], 3, 1, dil, dil);
        b.b[1] = bn(p + ".bn2", planes[L]);
      }
      b.has_ds = (i == 0) && ds;
      if (b.has_ds) {
        b.ds = conv(p + ".downsample.0", inplanes, out_c, 1, st, 0, 1);
        b.bd = bn(p + ".downsample.1", out_c);
      }
      s.blocks.push_back(b);
      inplanes = out_c;
      s.max_c = std::max(s.max_c, out_c);
    }
  }
  s.fc_cin = inplanes;
  add_entry(s.ptab, pc, "fc.weight", {D, inplanes, 1, 1}, &s.fc_w);
  add_entry(s.ptab, pc, "fc.bias", {D}, &s.fc_b);
  s.n_params = pc; s.n_buffers = bc;
  return s;
}

static bool arch_ok(int arch) { return arch == DDN_ARCH_RESNET34_8S || arch == DDN_ARCH_RESNET50_8S; }

static const NetSpec& get_spec(int arch, int D) {
  static std::mutex mu;
  static std::deque<NetSpec> cache;       // a deque: references handed out stay valid when it grows
  std::lock_guard<std::mutex> lk(mu);
  for (auto& s : cache) if (s.arch == arch && s.D == D) return s;
  cache.push_back(build_spec(arch, D));
  return cache.back();
}

// ------------------------------------------------------------------------------------------------ workspace plan
// mode: DDN_MODE_INFER (eval statistics, BatchNorm folded into the conv epilogues, nothing kept), DDN_MODE_TRAIN (batch
// statistics, activations kept for backward), DDN_MODE_EVAL_SAVE (frozen running statistics, activations kept: the reference
// backpropagates through an eval()-mode network this way).
struct ConvBufs { size_t raw, stats; int Hin, Win, Hout, Wout; };   // stats: [G][C] mean, then [G][C] 1/sqrt(var+eps)
struct PlaneBufs { size_t hi, lo; };   // bf16 operand planes of an activation (tensor-core modes only)
// act[j] / act_p[j]: relu(bn(c[j])) for j < n-1 (the input of c[j+1]); out / out_p: the block output
struct BlockBufs { ConvBufs c[3], ds; size_t act[2], out; PlaneBufs act_p[2], out_p; };
struct Plan {
  int arch, B, H, W, D, mode, precision;
  int H1, W1, Hp, Wp;
  size_t x4, stem_raw, stem_stats, pool_out, argmax;
  PlaneBufs pool_p, grad_p, patch_p;  // pooled stem output; current d(raw conv output); 7x7/2 stem patches [B,H1,W1,192]
  size_t wws;                         // packed-weight staging of the tensor-core convs
  bool tc;
  std::vector<BlockBufs> blk;
  size_t low, dlow;
  size_t wpack, wpack2, dwp, scratch[4];
  size_t fc_part;                     // fc_part_floats(C, D) floats: per-block partial sums of the fc gradient
  size_t acc, sums;                   // BatchNorm accumulator (bn_stats.cuh) and the backward's per-group sums
  size_t dwp_all;                     // [n_params + 64*192] doubles: every conv's [taps][Cout][Cin] gradient accumulator (tensor-core modes)
  size_t scratch_elems;
  size_t unit_dy;                     // DDN_NET_UNIT_DESCRIPTORS with a backward: [B, D, H, W] cotangent through the normalisation
  int flags;
  size_t total;
};

static float* stat_mean(char* ws, const ConvBufs& cb) { return reinterpret_cast<float*>(ws + cb.stats); }

static int make_plan(Plan* p, int arch, int B, int H, int W, int D, int mode, int precision, int flags = 0) {
  DDN_CHECK_ARG((flags & ~DDN_NET_UNIT_DESCRIPTORS) == 0, "unknown network flags 0x%x", flags);
  DDN_CHECK_ARG(arch_ok(arch), "unknown architecture id %d", arch);
  DDN_CHECK_ARG(B >= 1 && H >= 32 && W >= 32 && H % 8 == 0 && W % 8 == 0, "need B>=1 and H, W multiples of 8 (>=32); got B=%d H=%d W=%d", B, H, W);
  DDN_CHECK_ARG(D >= 1 && D <= 32, "descriptor dimension must be in [1,32] (got %d)", D);
  DDN_CHECK_ARG(precision >= DDN_PRECISION_FP32_SIMT && precision <= DDN_PRECISION_BF16, "unknown precision %d", precision);
  DDN_CHECK_ARG(mode >= DDN_MODE_INFER && mode <= DDN_MODE_EVAL_SAVE, "unknown mode %d", mode);
  const NetSpec& s = get_spec(arch, D);
  p->arch = arch; p->B = B; p->H = H; p->W = W; p->D = D; p->mode = mode; p->precision = precision;
  const int G = BN_MAX_GROUPS;
  size_t cur = 0;
  auto alloc = [&](size_t bytes) { size_t o = cur; cur += align_up(bytes, 256); return o; };
  auto f32 = [&](int64_t n) { return alloc(sizeof(float) * (size_t)n); };
  p->H1 = (H + 6 - 7) / 2 + 1; p->W1 = (W + 6 - 7) / 2 + 1;
  p->Hp = (p->H1 - 1) / 2 + 1; p->Wp = (p->W1 - 1) / 2 + 1;
  p->tc = precision != DDN_PRECISION_FP32_SIMT;
  p->x4 = p->tc ? 0 : f32((int64_t)B * H * W * 4);
  p->stem_raw = f32((int64_t)B * p->H1 * p->W1 * 64);
  p->stem_stats = f32(2 * G * 64);
  // fp32 pooled output: the SIMT instrument's activations, and the first residual of the folded inference path
  p->pool_out = (p->tc && mode != DDN_MODE_INFER) ? 0 : f32((int64_t)B * p->Hp * p->Wp * 64);
  p->argmax = alloc((size_t)B * p->Hp * p->Wp * 64);
  auto planes = [&](int64_t n) { PlaneBufs pb{0, 0}; if (p->tc) { pb.hi = alloc(2 * (size_t)n); pb.lo = alloc(2 * (size_t)n); } return pb; };
  p->pool_p = planes((int64_t)B * p->Hp * p->Wp * 64);
  p->patch_p = planes((int64_t)B * p->H1 * p->W1 * 192);
  int h = p->Hp, w = p->Wp;
  size_t max_w = 0;
  int64_t max_act = (int64_t)B * p->H1 * p->W1 * 64;
  int64_t max_up = 0;
  p->blk.clear();
  for (const BlockSpec& b : s.blocks) {
    BlockBufs bb;
    memset(&bb, 0, sizeof(bb));
    size_t blk_max_w = 0;
    auto conv_bufs = [&](const ConvSpec& c, int hin, int win) {
      ConvBufs cb; cb.Hin = hin; cb.Win = win;
      cb.Hout = (hin + 2 * c.pad - c.dil * (c.k - 1) - 1) / c.stride + 1;
      cb.Wout = (win + 2 * c.pad - c.dil * (c.k - 1) - 1) / c.stride + 1;
      cb.raw = f32((int64_t)B * cb.Hout * cb.Wout * c.cout);
      cb.stats = f32(2 * G * c.cout);
      blk_max_w = std::max(blk_max_w, (size_t)c.k * c.k * c.cin * c.cout);
      max_act = std::max(max_act, (int64_t)B * cb.Hout * cb.Wout * c.cout);
      // the data gradient of a strided conv zero-inserts dY [B, Hin, Win, Cout] into the gradient planes (only those)
      if (c.stride == 2) max_up = std::max(max_up, (int64_t)B * hin * win * c.cout);
      return cb;
    };
    const int last = b.n - 1;
    int hc = h, wc = w;
    for (int j = 0; j < b.n; ++j) {
      bb.c[j] = conv_bufs(b.c[j], hc, wc);
      hc = bb.c[j].Hout; wc = bb.c[j].Wout;
      const int64_t n_el = (int64_t)B * hc * wc * b.c[j].cout;
      // tensor-core modes keep activations only as bf16 hi/lo planes; the fp32 SIMT instrument keeps fp32 tensors
      if (j < last) {
        if (!p->tc) bb.act[j] = f32(n_el);
        bb.act_p[j] = planes(n_el);
      }
      if (j == last && b.has_ds) bb.ds = conv_bufs(b.ds, h, w);
    }
    if (!p->tc) bb.out = f32((int64_t)B * hc * wc * b.c[last].cout);
    bb.out_p = planes((int64_t)B * hc * wc * b.c[last].cout);
    // a tensor-core plan keeps no fp32 activations, so every block conv must have a tensor-core kernel (true for every H, W
    // accepted above; a change of the spec or of that rule becomes an error here instead of a null read in a SIMT conv)
    auto on_tc = [&](const ConvSpec& c, const ConvBufs& cb) { return tc_conv_supported(c.cin, c.cout, c.k, c.stride, c.pad, c.dil, cb.Hin, cb.Win); };
    bool all_tc = !b.has_ds || on_tc(b.ds, bb.ds);
    for (int j = 0; j < b.n; ++j) all_tc = all_tc && on_tc(b.c[j], bb.c[j]);
    if (p->tc && !all_tc) {
      set_error("a block convolution at %dx%d has no tensor-core kernel (precision %d)", h, w, precision);
      return DDN_EUNSUPPORTED;
    }
    // the packed weights of a conv without a cached pack are staged in a fixed-size area (conv_tc.cu)
    if (p->tc && blk_max_w > tc_max_weight_elems()) {
      set_error("a block convolution has %zu weights, more than the %zu the tensor-core weight staging holds", blk_max_w, tc_max_weight_elems());
      return DDN_EUNSUPPORTED;
    }
    max_w = std::max(max_w, blk_max_w);
    h = hc; w = wc;
    p->blk.push_back(bb);
  }
  DDN_CHECK_ARG(h * 8 == H && w * 8 == W, "internal: trunk output %dx%d is not H/8 x W/8", h, w);
  p->low = f32((int64_t)B * D * h * w);
  p->dlow = f32((int64_t)B * D * h * w);
  max_w = std::max(max_w, (size_t)7 * 7 * 4 * 64);
  p->wpack = f32((int64_t)max_w); p->wpack2 = f32((int64_t)max_w); p->dwp = f32((int64_t)max_w);
  p->acc = alloc(bn_accum_bytes(s.max_c));
  p->sums = f32(3 * 2 * G * s.max_c);     // [0]: standalone column-sum pass, [1], [2]: sums produced by a data-gradient epilogue
  p->scratch_elems = (size_t)max_act;
  for (int i = 0; i < 4; ++i) p->scratch[i] = f32((int64_t)max_act);
  p->grad_p = planes(std::max(max_act, max_up));
  p->wws = alloc(p->tc ? tc_weight_ws_bytes() : 0);
  p->dwp_all = (p->tc && mode != DDN_MODE_INFER) ? alloc(sizeof(double) * (size_t)(s.n_params + 64 * 192)) : 0;
  p->fc_part = mode != DDN_MODE_INFER ? f32((int64_t)fc_part_floats(s.fc_cin, D)) : 0;
  // last, so that a plan without the flag is byte for byte the plan of ddn_net_workspace_bytes
  p->flags = flags;
  p->unit_dy = ((flags & DDN_NET_UNIT_DESCRIPTORS) && mode != DDN_MODE_INFER) ? f32((int64_t)B * D * H * W) : 0;
  p->total = cur;
  return 0;
}

struct Ctx {
  const NetSpec* s; const Plan* p; char* ws; const float* params; float* buffers; float* grads;
  cudaStream_t st; float momentum, eps; int mode; int G;
  float* f(size_t off) const { return reinterpret_cast<float*>(ws + off); }
  double* d(size_t off) const { return reinterpret_cast<double*>(ws + off); }
  __nv_bfloat16* h(size_t off) const { return reinterpret_cast<__nv_bfloat16*>(ws + off); }
  TcPlanes planes(const PlaneBufs& b) const { return TcPlanes{h(b.hi), h(b.lo)}; }
  float* mean(size_t stats) const { return f(stats); }
  float* invstd(size_t stats, int C) const { return f(stats) + (size_t)G * C; }
  BnAccum accum() const { return bn_accum_at(ws + p->acc, s->max_c); }
  float* sums(int slot) const { return f(p->sums) + (size_t)slot * 2 * G * s->max_c; }
  bool training() const { return mode == DDN_MODE_TRAIN; }
};

// Optional caller-owned caches of the packed bf16 weights (forward and data-gradient packs of every conv), registered with
// ddn_resnet34_8s_set_weight_cache(), one slot per parameter array (two networks in one process do not evict each other).
// Validity is decided on the device: every forward fingerprints the parameter array and re-packs only when it changed
// (tc_pack_all), so no host-side version bookkeeping can go stale.  Layout: [tensor][forward | dgrad][hi | lo] at byte
// offset w_off * 8, then the two fingerprints in the last 256 bytes.
struct WeightCache {
  char* base = nullptr; size_t bytes = 0; uint64_t version = 0; const float* params = nullptr; int precision = -1;
  bool fresh = true;
};
static std::vector<WeightCache> g_wcaches;
static std::mutex g_wcache_mu;

static WeightCache* find_cache(const float* params) {
  for (auto& wc : g_wcaches) if (wc.params == params && wc.base) return &wc;
  return nullptr;
}
static size_t pack_offset(const ConvSpec& cs, int dgrad) {
  const size_t slot = (size_t)cs.cout * cs.cin * cs.k * cs.k;                 // the cache reserves 4 x numel bf16 per tensor
  return ((size_t)cs.w_off * 2 + (size_t)dgrad * slot) * 2 * sizeof(__nv_bfloat16);
}

// start of every tensor-core forward: make the cached packs match the parameters (3 launches; packs only when they changed)
static int ensure_packs(const Ctx& c) {
  std::lock_guard<std::mutex> lk(g_wcache_mu);
  WeightCache* wc = find_cache(c.params);
  if (!wc || wc->precision != c.p->precision) return 0;
  const NetSpec& s = *c.s;
  if (wc->bytes < (size_t)s.n_params * 8 + 512) { set_error("weight cache too small"); return DDN_EWORKSPACE; }
  std::vector<TcPackEntry> tab;
  auto add = [&](const ConvSpec& cs, int dgrad, int kind) {
    TcPackEntry e; e.w_off = cs.w_off; e.dst_off = (int64_t)pack_offset(cs, dgrad); e.Cout = cs.cout; e.Cin = cs.cin; e.k = cs.k;
    e.dgrad = dgrad; e.kind = kind;
    tab.push_back(e);
  };
  add(s.stem, 0, 1);
  for (const BlockSpec& b : s.blocks) {
    for (int j = 0; j < b.n; ++j) { add(b.c[j], 0, 0); add(b.c[j], 1, 0); }
    if (b.has_ds) { add(b.ds, 0, 0); add(b.ds, 1, 0); }
  }
  unsigned long long* fp_new = reinterpret_cast<unsigned long long*>(wc->base + wc->bytes - 256);
  unsigned long long* fp_old = reinterpret_cast<unsigned long long*>(wc->base + wc->bytes - 128);
  int force = 0;
  if (wc->fresh) {
    DDN_CUDA(cudaMemsetAsync(wc->base + wc->bytes - 256, 0, 256, c.st));
    force = 1; wc->fresh = false;
  }
  return tc_pack_all(c.params, s.n_params, wc->base, tab.data(), (int)tab.size(), fp_new, fp_old, force, c.p->precision, c.st);
}

// packed planes of conv `cs` (mode 0 = forward, 1 = data gradient; stem: [64][192] patch-GEMM layout) from the cache, or
// nullptr when no cache is registered for this parameter array (the conv then packs into the staging area per call)
static const TcPlanes* cached_pack(const Ctx& c, const ConvSpec& cs, int dgrad, TcPlanes* out) {
  std::lock_guard<std::mutex> lk(g_wcache_mu);
  WeightCache* wc = find_cache(c.params);
  if (!wc || wc->precision != c.p->precision || wc->fresh) return nullptr;
  const size_t wel = cs.k == 7 ? (size_t)64 * 192 : (size_t)cs.cout * cs.cin * cs.k * cs.k;
  __nv_bfloat16* hi = reinterpret_cast<__nv_bfloat16*>(wc->base + pack_offset(cs, dgrad));
  out->hi = hi; out->lo = hi + wel;
  return out;
}

// BatchNorm statistics request of a forward conv: batch statistics accumulated by the conv epilogue (training), or none
// (the statistics slots were filled from the running estimates by bn_eval_stats_all before the first conv)
static BnFwdFinal stats_request(const Ctx& c, const BnSpec& bs, const ConvBufs& cb, int64_t M) {
  BnFwdFinal f;
  f.a = c.accum();
  f.mean = c.mean(cb.stats); f.invstd = c.invstd(cb.stats, bs.C);
  f.running_mean = c.buffers + bs.rm_off; f.running_var = c.buffers + bs.rv_off;
  f.count = M / c.G; f.G = c.G; f.C = bs.C; f.momentum = c.momentum; f.eps = c.eps;
  return f;
}

// one conv (forward) + the statistics of the BatchNorm that follows it.
// Tensor-core convs read the bf16 planes of their input and accumulate the BN sums in their epilogue (the last CTA writes
// mean / invstd / running statistics); the fp32 SIMT convs read the fp32 tensor and the column sums come from a separate pass.
static int conv_bn_forward(const Ctx& c, const ConvSpec& cs, const BnSpec& bs, const float* in, const PlaneBufs& in_p,
                           const ConvBufs& cb, int N, int cin_eff) {
  const float* w = c.params + cs.w_off;
  float* raw = c.f(cb.raw);
  const int64_t M = (int64_t)N * cb.Hout * cb.Wout;
  const BnFwdFinal fin = stats_request(c, bs, cb, M);
  if (c.p->tc) {
    TcPlanes wpk_s; const TcPlanes* wpk = cached_pack(c, cs, 0, &wpk_s);
    return tc_conv_planes(c.planes(in_p), w, wpk, raw, nullptr, c.training() ? &fin : nullptr, N, cb.Hin, cb.Win, cs.cin, cs.cout, cs.k,
                          cs.stride, cs.dil, 0, c.p->precision, c.ws + c.p->wws, tc_weight_ws_bytes(), c.st);
  }
  ConvGeom g;
  DDN_TRY(conv_geom_init(&g, N, cb.Hin, cb.Win, cin_eff, cb.Hout, cb.Wout, cs.cout, cs.k, cs.k, cs.stride, 1, cs.pad, cs.dil));
  DDN_TRY(launch_pack_weights(w, c.f(c.p->wpack), cs.cout, cs.cin, cin_eff, cs.k, cs.k, 0, c.st));
  {
    ProfScope ps(PROF_CONV_FWD_SIMT, 2.0 * M * (double)cs.cout * cs.k * cs.k * cs.cin, c.st);
    DDN_TRY(launch_conv_gather_f32(in, c.f(c.p->wpack), nullptr, raw, g, c.st));
  }
  if (c.training())
    return launch_bn_stats(raw, M, bs.C, c.G, fin.a, fin.mean, fin.invstd, fin.running_mean, fin.running_var, c.momentum, c.eps, c.st);
  return 0;
}

// Inference (eval-mode BN) on the tensor-core path: BN is a per-channel multiply-add of the conv accumulator, so the conv
// epilogue applies it together with the residual add and the ReLU and writes the next conv's operand planes itself; no
// un-normalised conv output and no separate BN pass exist.  `out` / `out_p` may be absent (null / {0,0}).
static int conv_bn_folded(const Ctx& c, const ConvSpec& cs, const BnSpec& bs, const PlaneBufs& in_p, const ConvBufs& cb, int N,
                          float* out, const PlaneBufs* out_p, const float* addend, int relu) {
  float* scale = c.f(cb.stats); float* shift = c.f(cb.stats) + bs.C;     // the per-conv statistics slots hold scale / shift here
  DDN_TRY(launch_bn_fold(c.buffers + bs.rm_off, c.buffers + bs.rv_off, c.params + bs.g_off, c.params + bs.b_off, bs.C, c.eps,
                         scale, shift, c.st));
  TcPlanes wpk_s; const TcPlanes* wpk = cached_pack(c, cs, 0, &wpk_s);
  TcFoldedEpilogue ep = {scale, shift, relu, out_p ? c.h(out_p->hi) : nullptr, out_p ? c.h(out_p->lo) : nullptr};
  return tc_conv_planes(c.planes(in_p), c.params + cs.w_off, wpk, out, addend, nullptr, N, cb.Hin, cb.Win, cs.cin, cs.cout, cs.k,
                        cs.stride, cs.dil, 0, c.p->precision, c.ws + c.p->wws, tc_weight_ws_bytes(), c.st, &ep);
}

// every BatchNorm's statistics slots <- running estimates, in one launch (modes without batch statistics)
static int fill_eval_stats(const Ctx& c) {
  const NetSpec& s = *c.s; const Plan& p = *c.p;
  std::vector<BnEvalSeg> segs;
  auto add = [&](const BnSpec& bs, size_t stats_off) {
    BnEvalSeg sg; sg.rm_off = bs.rm_off; sg.rv_off = bs.rv_off; sg.stat_off = (int64_t)(stats_off / sizeof(float)); sg.C = bs.C;
    segs.push_back(sg);
  };
  add(s.stem_bn, p.stem_stats);
  for (size_t i = 0; i < s.blocks.size(); ++i) {
    for (int j = 0; j < s.blocks[i].n; ++j) add(s.blocks[i].b[j], p.blk[i].c[j].stats);
    if (s.blocks[i].has_ds) add(s.blocks[i].bd, p.blk[i].ds.stats);
  }
  return launch_bn_eval_stats_all(c.buffers, reinterpret_cast<float*>(c.ws), segs.data(), (int)segs.size(), c.G, c.eps, c.st);
}

static int net_forward(const Ctx& c, const float* x, float* y, float* low_nhwc) {
  const NetSpec& s = *c.s; const Plan& p = *c.p;
  const int B = p.B, G = c.G;
  const bool want_lo = p.precision == DDN_PRECISION_BF16X3;
  const bool fold = c.mode == DDN_MODE_INFER && p.tc;
  DDN_CUDA(cudaMemsetAsync(c.ws + p.acc, 0, bn_accum_bytes(s.max_c), c.st));     // the workspace arrives uninitialised
  if (p.tc) DDN_TRY(ensure_packs(c));
  if (!c.training() && !fold) DDN_TRY(fill_eval_stats(c));
  // stem: conv1 7x7/2 -> bn1 -> relu -> maxpool 3x3/2          (resnet.py:232-235)
  ConvBufs stem_cb{p.stem_raw, p.stem_stats, p.H, p.W, p.H1, p.W1};
  if (p.tc) {   // conv1 as a K = 192 GEMM over 7x7/2 patch planes, BN statistics from the conv epilogue
    DDN_TRY(tc_stem_patches(x, c.h(p.patch_p.hi), c.h(p.patch_p.lo), B, p.H, p.W, p.precision, c.st));
    const BnFwdFinal fin = stats_request(c, s.stem_bn, stem_cb, (int64_t)B * p.H1 * p.W1);
    TcPlanes wpk_s; const TcPlanes* wpk = cached_pack(c, s.stem, 0, &wpk_s);
    DDN_TRY(tc_stem_forward(c.planes(p.patch_p), c.params + s.stem.w_off, wpk, c.f(p.stem_raw), c.training() ? &fin : nullptr, B, p.H1,
                            p.W1, p.precision, c.ws + p.wws, tc_weight_ws_bytes(), c.st));
    if (fold) DDN_TRY(launch_bn_eval_stats(c.buffers + s.stem_bn.rm_off, c.buffers + s.stem_bn.rv_off, 64, G, c.eps,
                                           c.mean(p.stem_stats), c.invstd(p.stem_stats, 64), c.st));
  } else {
    DDN_TRY(launch_nchw_to_nhwc4(x, c.f(p.x4), B, p.H, p.W, c.st));
    DDN_TRY(conv_bn_forward(c, s.stem, s.stem_bn, c.f(p.x4), PlaneBufs{0, 0}, stem_cb, B, 4));
  }
  DDN_TRY(launch_stem_bn_relu_pool(c.f(p.stem_raw), c.mean(p.stem_stats), c.invstd(p.stem_stats, 64), c.params + s.stem_bn.g_off,
                                   c.params + s.stem_bn.b_off, (p.tc && c.mode != DDN_MODE_INFER) ? nullptr : c.f(p.pool_out), reinterpret_cast<uint8_t*>(c.ws + p.argmax),
                                   p.tc ? c.h(p.pool_p.hi) : nullptr, (p.tc && want_lo) ? c.h(p.pool_p.lo) : nullptr,
                                   B, p.H1, p.W1, 64, G, c.st));
  const float* cur = p.tc ? nullptr : c.f(p.pool_out);      // fp32 activations exist only in the SIMT instrument
  PlaneBufs cur_p = p.pool_p;
  for (size_t i = 0; i < s.blocks.size(); ++i) {        // BasicBlock.forward, resnet.py:53-69 / Bottleneck.forward, :87-109
    const BlockSpec& b = s.blocks[i]; const BlockBufs& bb = p.blk[i];
    const int last = b.n - 1;
    if (fold) {
      PlaneBufs in_p = cur_p;
      for (int j = 0; j < last; ++j) {     // act[j]: planes only
        DDN_TRY(conv_bn_folded(c, b.c[j], b.b[j], in_p, bb.c[j], B, nullptr, &bb.act_p[j], nullptr, 1));
        in_p = bb.act_p[j];
      }
      // the epilogue's residual addend is fp32: the pooled stem output for the first block, else the previous block's fp32
      // output, which the folded path keeps in that block's (otherwise unused) last raw slot
      const float* res = i == 0 ? c.f(p.pool_out) : c.f(p.blk[i - 1].c[last].raw);
      if (b.has_ds) {
        DDN_TRY(conv_bn_folded(c, b.ds, b.bd, cur_p, bb.ds, B, c.f(bb.ds.raw), nullptr, nullptr, 0));  // bn_d(conv_d(x)), fp32
        res = c.f(bb.ds.raw);
      }
      DDN_TRY(conv_bn_folded(c, b.c[last], b.b[last], in_p, bb.c[last], B, c.f(bb.c[last].raw), &bb.out_p, res, 1));   // fp32 block output
      cur = c.f(bb.c[last].raw);
      cur_p = bb.out_p;
      continue;
    }
    const float* in = cur; PlaneBufs in_p = cur_p;
    for (int j = 0; j < last; ++j) {       // act[j] = relu(bn_j(conv_j(in)))
      DDN_TRY(conv_bn_forward(c, b.c[j], b.b[j], in, in_p, bb.c[j], B, b.c[j].cin));
      BnApplyArgs a1;
      memset(&a1, 0, sizeof(a1));
      a1.x = c.f(bb.c[j].raw); a1.mean = c.mean(bb.c[j].stats); a1.invstd = c.invstd(bb.c[j].stats, b.b[j].C);
      a1.gamma = c.params + b.b[j].g_off; a1.beta = c.params + b.b[j].b_off;
      a1.y = p.tc ? nullptr : c.f(bb.act[j]); a1.hi = p.tc ? c.h(bb.act_p[j].hi) : nullptr;
      a1.lo = (p.tc && want_lo) ? c.h(bb.act_p[j].lo) : nullptr;
      a1.M = (int64_t)B * bb.c[j].Hout * bb.c[j].Wout; a1.C = b.b[j].C; a1.relu = 1; a1.G = G;
      DDN_TRY(launch_bn_apply(a1, c.st));
      in = p.tc ? nullptr : c.f(bb.act[j]); in_p = bb.act_p[j];
    }
    DDN_TRY(conv_bn_forward(c, b.c[last], b.b[last], in, in_p, bb.c[last], B, b.c[last].cin));
    BnApplyArgs a2;
    memset(&a2, 0, sizeof(a2));
    a2.x = c.f(bb.c[last].raw); a2.mean = c.mean(bb.c[last].stats); a2.invstd = c.invstd(bb.c[last].stats, b.b[last].C);
    a2.gamma = c.params + b.b[last].g_off; a2.beta = c.params + b.b[last].b_off;
    a2.y = p.tc ? nullptr : c.f(bb.out); a2.hi = p.tc ? c.h(bb.out_p.hi) : nullptr; a2.lo = (p.tc && want_lo) ? c.h(bb.out_p.lo) : nullptr;
    a2.M = (int64_t)B * bb.c[last].Hout * bb.c[last].Wout; a2.C = b.b[last].C; a2.relu = 1; a2.G = G;
    if (b.has_ds) {
      DDN_TRY(conv_bn_forward(c, b.ds, b.bd, cur, cur_p, bb.ds, B, b.ds.cin));
      a2.r = c.f(bb.ds.raw); a2.rmean = c.mean(bb.ds.stats); a2.rinvstd = c.invstd(bb.ds.stats, b.bd.C);
      a2.rgamma = c.params + b.bd.g_off; a2.rbeta = c.params + b.bd.b_off;
    } else if (p.tc) {           // identity residual straight from the block input's operand planes
      a2.r_hi = c.h(cur_p.hi); a2.r_lo = want_lo ? c.h(cur_p.lo) : nullptr;
    } else {
      a2.r = cur;
    }
    DDN_TRY(launch_bn_apply(a2, c.st));
    cur = p.tc ? nullptr : c.f(bb.out);
    cur_p = bb.out_p;
  }
  // fc (1x1 conv + bias) and the bilinear upsample back to the input size      (resnet.py:263, resnet_dilated.py:320)
  const int h8 = p.H / 8, w8 = p.W / 8;
  const bool feat_planes = p.tc;       // the features are read from the operand planes (hi + lo)
  DDN_TRY(launch_fc_forward(feat_planes ? nullptr : cur, feat_planes ? c.h(cur_p.hi) : nullptr,
                            (feat_planes && want_lo) ? c.h(cur_p.lo) : nullptr, c.params + s.fc_w, c.params + s.fc_b, c.f(p.low),
                            low_nhwc, (int64_t)h8 * w8, B, s.fc_cin, p.D, c.st));
  if (p.flags & DDN_NET_UNIT_DESCRIPTORS)    // y = x / ||x|| per pixel (dense_correspondence_network.py:256-259)
    DDN_TRY(launch_upsample_unit_fwd(c.f(p.low), y, B, p.D, h8, w8, p.H, p.W, c.st));
  else
    DDN_TRY(launch_upsample_fwd(c.f(p.low), y, B * p.D, h8, w8, p.H, p.W, c.st));
  return 0;
}

// fp32 SIMT weight gradient of one conv: dw [Cout][Cin][k][k] (overwritten) through the zero-filled packed scratch `dwp`
// [k*k*cin_eff*Cout] (cin_eff = Cin padded to the gather's channel count: 4 for the stem's NHWC4 image)
static int simt_wgrad(const float* in, const float* dy, float* dwp, float* dw, int N, int Hin, int Win, int cin, int cin_eff, int Hout,
                      int Wout, int cout, int k, int stride, int pad, int dil, cudaStream_t st) {
  ConvGeom g;
  DDN_TRY(conv_geom_init(&g, N, Hin, Win, cin_eff, Hout, Wout, cout, k, k, stride, 1, pad, dil));
  DDN_TRY(launch_fill_zero(dwp, sizeof(float) * (size_t)k * k * cin_eff * cout, st));
  {
    ProfScope ps(PROF_CONV_WGRAD_SIMT, 2.0 * N * Hout * Wout * (double)cout * k * k * cin, st);
    DDN_TRY(launch_conv_wgrad_f32(in, dy, dwp, g, st));
  }
  return launch_unpack_wgrad(dwp, dw, cout, cin, cin_eff, k, k, st);
}

// conv backward: dw -> grads (SIMT: immediately; tensor core: accumulated in dwp_all, converted per bucket), dx -> `dx`
// (+ addend) when dx != nullptr.  Tensor-core convs take the saved bf16 planes of their input and the planes of dY
// (p.grad_p, written by the BN backward that precedes this call); the fp32 SIMT convs take the fp32 tensors.
static int conv_backward(const Ctx& c, const ConvSpec& cs, const float* in, const PlaneBufs& in_p, const float* dy, float* dx,
                         const float* addend, int N, int Hin, int Win, int Hout, int Wout, int cin_eff, const TcBwdStats* bst = nullptr) {
  const Plan& p = *c.p;
  const float* w = c.params + cs.w_off;
  float* dw = c.grads + cs.w_off;
  const double fl = 2.0 * N * Hout * Wout * (double)cs.cout * cs.k * cs.k * cs.cin;
  if (p.tc) {
    DDN_TRY(tc_wgrad_planes(c.planes(in_p), c.planes(p.grad_p), nullptr, N, Hin, Win, cs.cin, cs.cout, cs.k, cs.stride, cs.dil,
                            p.precision, c.d(p.dwp_all) + cs.w_off, c.st));
    if (dx) {
      TcPlanes wpk_s; const TcPlanes* wpk = cached_pack(c, cs, 1, &wpk_s);
      if (cs.stride == 2)   // zero-insert the fp32 dY into the (now free) gradient planes, then an ordinary stride-1 dgrad
        DDN_TRY(tc_dgrad_strided(dy, c.planes(p.grad_p), w, wpk, dx, addend, N, Hin, Win, cs.cin, cs.cout, cs.k, p.precision,
                                 c.ws + p.wws, tc_weight_ws_bytes(), c.st, bst));
      else
        DDN_TRY(tc_conv_planes(c.planes(p.grad_p), w, wpk, dx, addend, nullptr, N, Hin, Win, cs.cin, cs.cout, cs.k, 1, cs.dil, 1,
                               p.precision, c.ws + p.wws, tc_weight_ws_bytes(), c.st, nullptr, bst));
    }
    return 0;
  }
  DDN_CHECK_ARG(bst == nullptr, "backward statistics can only ride on a tensor-core data gradient");
  DDN_TRY(simt_wgrad(in, dy, c.f(p.dwp), dw, N, Hin, Win, cs.cin, cin_eff, Hout, Wout, cs.cout, cs.k, cs.stride, cs.pad, cs.dil, c.st));
  if (dx) {
    ConvGeom gd;
    DDN_TRY(conv_geom_init(&gd, N, Hout, Wout, cs.cout, Hin, Win, cs.cin, cs.k, cs.k, 1, cs.stride, cs.dil * (cs.k - 1) - cs.pad, cs.dil));
    DDN_TRY(launch_pack_weights(w, c.f(p.wpack2), cs.cout, cs.cin, cs.cin, cs.k, cs.k, 1, c.st));
    ProfScope ps(PROF_CONV_DGRAD_SIMT, fl, c.st);
    DDN_TRY(launch_conv_gather_f32(dy, c.f(p.wpack2), addend, dx, gd, c.st));
  }
  return 0;
}

// BN backward of `bs` (output y = relu?(bn(raw) + res)) whose dx feeds conv `cs`'s backward: planes for a tensor-core conv,
// fp32 for a SIMT conv.  mask: the bf16 hi plane of y / the fp32 y / recomputed from raw (no residual) -- see BnBwdArgs.
// fused_slot > 0: the column sums were produced by the data-gradient epilogue that wrote `dy` (bwd_stats_for) -- skip that pass.
static int bn_backward_for(const Ctx& c, const BnSpec& bs, const ConvBufs& cb, const float* dy, const float* y_f32,
                           const __nv_bfloat16* y_hi, int relu, float* g_out, const ConvSpec& cs, float* dx_f32, int64_t M,
                           int fused_slot = 0) {
  BnBwdArgs a;
  memset(&a, 0, sizeof(a));
  a.dy = dy; a.x = c.f(cb.raw); a.mean = c.mean(cb.stats); a.invstd = c.invstd(cb.stats, bs.C);
  a.gamma = c.params + bs.g_off; a.beta = c.params + bs.b_off;
  a.y = y_f32; a.y_hi = y_hi; a.g_out = g_out;
  a.dgamma = c.grads + bs.g_off; a.dbeta = c.grads + bs.b_off;
  a.acc = c.accum(); a.sums = c.sums(fused_slot);
  a.sums_ready = fused_slot > 0;
  a.M = M; a.C = bs.C; a.relu = relu; a.training = c.training() ? 1 : 0; a.G = c.G;
  if (c.p->tc) {
    a.dx = cs.stride == 2 ? dx_f32 : nullptr;      // the strided data gradient re-reads dY in fp32 (zero insertion)
    a.dx_hi = c.h(c.p->grad_p.hi);
    a.dx_lo = c.p->precision == DDN_PRECISION_BF16X3 ? c.h(c.p->grad_p.lo) : nullptr;
  } else {
    a.dx = dx_f32;
  }
  return launch_bn_backward(a, c.st);
}

// Column sums of BatchNorm `bs` (y = relu(bn(raw) [+ residual])) computed by the epilogue of the tensor-core data gradient that
// produces its dY (conv_tc.cuh TcBwdStats) instead of a separate pass over dY and raw.
static bool bwd_stats_for(const Ctx& c, const BnSpec& bs, const ConvBufs& cb, const __nv_bfloat16* y_hi, int slot, TcBwdStats* out) {
  if (!c.p->tc) return false;
  memset(out, 0, sizeof(*out));
  out->raw = c.f(cb.raw); out->y_hi = y_hi; out->mean = c.mean(cb.stats); out->invstd = c.invstd(cb.stats, bs.C);
  out->gamma = c.params + bs.g_off; out->beta = c.params + bs.b_off; out->relu = 1;
  out->fin.a = c.accum(); out->fin.sums = c.sums(slot);
  out->fin.dgamma = c.grads + bs.g_off; out->fin.dbeta = c.grads + bs.b_off; out->fin.G = c.G; out->fin.C = bs.C;
  return true;
}

// The stem's backward: maxpool -> relu -> bn1 -> conv1 (weight gradient only; the image is not differentiated).  net_backward
// runs it on its workspace, ddn_stem_backward on caller tensors.
struct StemBwdArgs {
  const float* dy_pool; const uint8_t* argmax;                       // [N,Hp,Wp,64]
  const float* raw; const float* mean; const float* invstd;          // raw [N,H1,W1,64], statistics [G][64]
  const float* gamma; const float* beta; float* dgamma; float* dbeta;
  float* g;                       // [N,H1,W1,64]: the pre-BatchNorm gradient d(relu out) * (bn(raw) > 0)
  float* dx;                      // [N,H1,W1,64]: d raw in fp32 -- the SIMT conv's dY; optional on the tensor cores
  BnAccum acc; float* sums;       // BatchNorm-backward accumulator (zero) and [G][2][64] floats
  // tensor cores: the 7x7/2 patch planes of the image, the planes of d raw, and the pre-zeroed fp64 [64][192] accumulator the
  // caller converts (stem_unpack_entry)
  TcPlanes patches; __nv_bfloat16* dx_hi; __nv_bfloat16* dx_lo; double* dwp;
  // FP32_SIMT: the NHWC4 image, 7*7*4*64 floats of scratch, the conv1.weight gradient [64][3][7][7]
  const float* x4; float* dwp_f32; float* dw;
  int N, H, W, H1, W1, G, training, precision;
};

static int stem_backward(const StemBwdArgs& a, cudaStream_t st) {
  DDN_TRY(launch_stem_pool_relu_backward(a.dy_pool, a.argmax, a.raw, a.mean, a.invstd, a.gamma, a.beta, a.g, a.N, a.H1, a.W1, 64, a.G, st));
  const bool tc = a.precision != DDN_PRECISION_FP32_SIMT;
  BnBwdArgs ks;
  memset(&ks, 0, sizeof(ks));
  ks.dy = a.g; ks.x = a.raw; ks.mean = a.mean; ks.invstd = a.invstd; ks.gamma = a.gamma; ks.beta = a.beta;
  ks.dgamma = a.dgamma; ks.dbeta = a.dbeta; ks.acc = a.acc; ks.sums = a.sums;
  ks.M = (int64_t)a.N * a.H1 * a.W1; ks.C = 64; ks.relu = 0; ks.training = a.training; ks.G = a.G;
  ks.dx = a.dx;
  if (tc) { ks.dx_hi = a.dx_hi; ks.dx_lo = a.precision == DDN_PRECISION_BF16X3 ? a.dx_lo : nullptr; }
  DDN_TRY(launch_bn_backward(ks, st));
  if (tc) return tc_stem_wgrad(a.patches, TcPlanes{a.dx_hi, a.dx_lo}, a.N, a.H1, a.W1, a.precision, a.dwp, st);
  return simt_wgrad(a.x4, a.dx, a.dwp_f32, a.dw, a.N, a.H, a.W, 3, 4, a.H1, a.W1, 64, 7, 2, 3, 1, st);
}

// the conversion of the stem's [64][192] fp64 accumulator at dwp_base + src_off to conv1.weight at grads_base + dst_off
static TcUnpackEntry stem_unpack_entry(int64_t src_off, int64_t dst_off) {
  TcUnpackEntry e; e.src_off = src_off; e.dst_off = dst_off; e.Cout = 64; e.Cin = 3; e.taps = 49; e.kind = 1;
  return e;
}

// gradient buckets, in the order the backward completes them (ddn_grad_bucket_fn): [first block of the layer .. next bucket)
struct Bucket { int64_t begin, end; };

static int net_backward(const Ctx& c, const float* dy, const float* dlow_nhwc, ddn_grad_bucket_fn on_bucket, void* user) {
  const NetSpec& s = *c.s; const Plan& p = *c.p;
  const int B = p.B, h8 = p.H / 8, w8 = p.W / 8;
  const bool want_lo = p.precision == DDN_PRECISION_BF16X3;
  float* S[4] = {c.f(p.scratch[0]), c.f(p.scratch[1]), c.f(p.scratch[2]), c.f(p.scratch[3])};
  DDN_CUDA(cudaMemsetAsync(c.ws + p.acc, 0, bn_accum_bytes(s.max_c), c.st));
  if (p.tc) DDN_CUDA(cudaMemsetAsync(c.d(p.dwp_all), 0, sizeof(double) * (size_t)(s.n_params + 64 * 192), c.st));
  const BlockBufs& last = p.blk.back();
  // d(low) = upsample^T(dy) [+ the gradient the fused loss scattered straight into the low-resolution map]
  // (unit descriptors: dy first goes through the normalisation's Jacobian; dlow_nhwc already has, in the fused loss)
  if (dy && (p.flags & DDN_NET_UNIT_DESCRIPTORS))
    DDN_TRY(launch_upsample_unit_bwd(c.f(p.low), dy, c.f(p.dlow), c.f(p.unit_dy), B, p.D, h8, w8, p.H, p.W, c.st));
  else if (dy)
    DDN_TRY(launch_upsample_bwd(dy, c.f(p.dlow), B * p.D, h8, w8, p.H, p.W, c.st));
  if (dlow_nhwc) DDN_TRY(launch_add_lowres_nhwc(dlow_nhwc, c.f(p.dlow), (int64_t)h8 * w8, B, p.D, dy ? 1 : 0, c.st));
  int cur = 0;   // index of the scratch buffer holding d(block output)
  DDN_TRY(launch_fc_backward(c.f(p.dlow), p.tc ? nullptr : c.f(last.out), p.tc ? c.h(last.out_p.hi) : nullptr,
                             (p.tc && want_lo) ? c.h(last.out_p.lo) : nullptr, c.params + s.fc_w, S[cur], c.grads + s.fc_w,
                             c.grads + s.fc_b, c.f(p.fc_part), (int64_t)h8 * w8, B, s.fc_cin, p.D, c.st));
  std::vector<TcUnpackEntry> pending;      // tensor-core weight gradients waiting in dwp_all for the bucket's conversion
  auto defer = [&](const ConvSpec& cs) {
    if (!p.tc) return;
    TcUnpackEntry e; e.src_off = cs.w_off; e.dst_off = cs.w_off; e.Cout = cs.cout; e.Cin = cs.cin; e.taps = cs.k * cs.k; e.kind = 0;
    pending.push_back(e);
  };
  int64_t bucket_end = s.n_params;
  int bucket_id = 0;
  struct WindowGuard { ~WindowGuard() { g_window_reserved.store(0, std::memory_order_relaxed); } } window_guard;
  auto close_bucket = [&](int64_t begin) -> int {
    if (!pending.empty()) DDN_TRY(tc_unpack_wgrads(pending.data(), (int)pending.size(), c.d(p.dwp_all), c.grads, c.st));
    pending.clear();
    if (on_bucket) {
      on_bucket(user, bucket_id, begin, bucket_end - begin);
      g_window_reserved.store(overlap_window_sms(), std::memory_order_relaxed);     // a collective is in flight from here on
    }
    ++bucket_id; bucket_end = begin;
    return 0;
  };
  bool out_fused = false;   // the column sums of this block's last BatchNorm came out of the next block's conv1 data gradient (slot 2)
  for (int i = (int)s.blocks.size() - 1; i >= 0; --i) {
    const BlockSpec& b = s.blocks[i]; const BlockBufs& bb = p.blk[i];
    const int last = b.n - 1;
    const float* xin = p.tc ? nullptr : (i == 0 ? c.f(p.pool_out) : c.f(p.blk[i - 1].out));
    const PlaneBufs xin_p = i == 0 ? p.pool_p : p.blk[i - 1].out_p;
    auto rows = [&](const ConvBufs& cb) { return (int64_t)B * cb.Hout * cb.Wout; };
    int t1 = (cur + 1) & 3, t2 = (cur + 2) & 3, t3 = (cur + 3) & 3;
    // out = relu(bn_last(raw_last) + residual):  g = dOut*(out>0) -> S[t2];  d raw_last -> planes (tensor core) or S[t1] (fp32)
    DDN_TRY(bn_backward_for(c, b.b[last], bb.c[last], S[cur], p.tc ? nullptr : c.f(bb.out), p.tc ? c.h(bb.out_p.hi) : nullptr, 1, S[t2],
                            b.c[last], S[t1], rows(bb.c[last]), out_fused ? 2 : 0));
    // conv_j (j = last .. 1): dW, d act[j-1] -> S[t3] (+ the column sums of bn_{j-1}'s backward, in the same epilogue); then
    // act[j-1] = relu(bn_{j-1}(raw)), no residual: the mask is recomputed from raw in the tensor-core modes
    TcBwdStats st_in, st_next;
    bool in_fused = false;
    for (int j = last; j >= 1; --j) {
      in_fused = bwd_stats_for(c, b.b[j - 1], bb.c[j - 1], nullptr, 1, &st_in);
      DDN_TRY(conv_backward(c, b.c[j], p.tc ? nullptr : c.f(bb.act[j - 1]), bb.act_p[j - 1], S[t1], S[t3], nullptr, B, bb.c[j].Hin,
                            bb.c[j].Win, bb.c[j].Hout, bb.c[j].Wout, b.c[j].cin, in_fused ? &st_in : nullptr));
      defer(b.c[j]);
      if (j > 1)
        DDN_TRY(bn_backward_for(c, b.b[j - 1], bb.c[j - 1], S[t3], p.tc ? nullptr : c.f(bb.act[j - 1]), nullptr, 1, nullptr, b.c[j - 1],
                                S[t1], rows(bb.c[j - 1]), in_fused ? 1 : 0));
    }
    // conv1's data gradient completes d(block input) = dOut of the previous block: that block's last BatchNorm gets its column
    // sums there
    out_fused = i > 0 && bwd_stats_for(c, s.blocks[i - 1].b[last], p.blk[i - 1].c[last], c.h(p.blk[i - 1].out_p.hi), 2, &st_next);
    if (!b.has_ds) {
      DDN_TRY(bn_backward_for(c, b.b[0], bb.c[0], S[t3], p.tc ? nullptr : c.f(bb.act[0]), nullptr, 1, nullptr, b.c[0], S[t1],
                              rows(bb.c[0]), in_fused ? 1 : 0));
      // dX = dgrad(conv1) + g
      DDN_TRY(conv_backward(c, b.c[0], xin, xin_p, S[t1], S[t3], S[t2], B, bb.c[0].Hin, bb.c[0].Win, bb.c[0].Hout, bb.c[0].Wout, b.c[0].cin,
                            out_fused ? &st_next : nullptr));
      defer(b.c[0]);
      cur = t3;
    } else {
      // residual branch first (its dY planes are consumed before conv1's overwrite them):
      // bn_d(raw_d): d raw_d; ds conv: dW, dX_ds -> S[cur]
      DDN_TRY(bn_backward_for(c, b.bd, bb.ds, S[t2], nullptr, nullptr, 0, nullptr, b.ds, S[t1], rows(bb.ds)));
      DDN_TRY(conv_backward(c, b.ds, xin, xin_p, S[t1], S[cur], nullptr, B, bb.ds.Hin, bb.ds.Win, bb.ds.Hout, bb.ds.Wout, b.ds.cin));
      defer(b.ds);
      // main branch: d raw1, then dX = dgrad(conv1) + dX_ds -> S[t2]
      DDN_TRY(bn_backward_for(c, b.b[0], bb.c[0], S[t3], p.tc ? nullptr : c.f(bb.act[0]), nullptr, 1, nullptr, b.c[0], S[t1],
                              rows(bb.c[0]), in_fused ? 1 : 0));
      DDN_TRY(conv_backward(c, b.c[0], xin, xin_p, S[t1], S[t2], S[cur], B, bb.c[0].Hin, bb.c[0].Win, bb.c[0].Hout, bb.c[0].Wout, b.c[0].cin,
                            out_fused ? &st_next : nullptr));
      defer(b.c[0]);
      cur = t2;
      // a block with a downsample branch opens a residual layer: everything from its first parameter up is final now
      // (layer4 (+fc), layer3, layer2; layer1 -- whose first block has a downsample in the Bottleneck network -- and the stem
      // close together at the end)
      if (i > 0) DDN_TRY(close_bucket(b.c[0].w_off));
    }
  }
  // stem: maxpool -> relu -> bn1 -> conv1
  StemBwdArgs sa;
  memset(&sa, 0, sizeof(sa));
  sa.dy_pool = S[cur]; sa.argmax = reinterpret_cast<const uint8_t*>(c.ws + p.argmax);
  sa.raw = c.f(p.stem_raw); sa.mean = c.mean(p.stem_stats); sa.invstd = c.invstd(p.stem_stats, 64);
  sa.gamma = c.params + s.stem_bn.g_off; sa.beta = c.params + s.stem_bn.b_off;
  sa.dgamma = c.grads + s.stem_bn.g_off; sa.dbeta = c.grads + s.stem_bn.b_off;
  sa.g = S[(cur + 1) & 3]; sa.acc = c.accum(); sa.sums = c.f(p.sums);
  sa.N = B; sa.H = p.H; sa.W = p.W; sa.H1 = p.H1; sa.W1 = p.W1; sa.G = c.G; sa.training = c.training() ? 1 : 0; sa.precision = p.precision;
  if (p.tc) {
    sa.patches = c.planes(p.patch_p); sa.dx_hi = c.h(p.grad_p.hi); sa.dx_lo = c.h(p.grad_p.lo); sa.dwp = c.d(p.dwp_all) + s.n_params;
  } else {
    sa.dx = S[(cur + 2) & 3]; sa.x4 = c.f(p.x4); sa.dwp_f32 = c.f(p.dwp); sa.dw = c.grads + s.stem.w_off;
  }
  DDN_TRY(stem_backward(sa, c.st));
  if (p.tc) pending.push_back(stem_unpack_entry(s.n_params, s.stem.w_off));
  return close_bucket(0);
}

}  // namespace ddn

using namespace ddn;

extern "C" int ddn_abi_version(void) { return DDN_ABI_VERSION; }
extern "C" int ddn_set_reserved_sms(int n) {
  DDN_CHECK_ARG(n >= 0 && n <= 64, "reserved SM count must be in [0, 64]");
  g_reserved_sms.store(n);
  return 0;
}
extern "C" const char* ddn_last_error(void) { return g_err; }
extern "C" int64_t ddn_kernel_launch_count(void) { return g_launches.load(); }

extern "C" int ddn_profile_enable(int on) { g_prof_on.store(on ? 1 : 0); return 0; }
extern "C" int ddn_profile_reset(void) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  g_prof_used = 0;
  return 0;
}
extern "C" int ddn_profile_read(ddn_profile_entry* out, int cap) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  double ms[PROF_NUM_CLASSES] = {0}, work[PROF_NUM_CLASSES] = {0};
  int64_t n[PROF_NUM_CLASSES] = {0};
  for (size_t i = 0; i < g_prof_used; ++i) {
    float t = 0.f;
    if (cudaEventSynchronize(g_prof[i].b) != cudaSuccess || cudaEventElapsedTime(&t, g_prof[i].a, g_prof[i].b) != cudaSuccess) continue;
    ms[g_prof[i].cls] += t; work[g_prof[i].cls] += g_prof[i].work; n[g_prof[i].cls]++;
  }
  int k = 0;
  for (int c = 0; c < PROF_NUM_CLASSES; ++c) {
    if (!n[c]) continue;
    if (out && k < cap) {
      memset(&out[k], 0, sizeof(out[k]));
      snprintf(out[k].name, sizeof(out[k].name), "%s", kProfNames[c]);
      out[k].launches = n[c]; out[k].ms = ms[c]; out[k].work = work[c];
    }
    ++k;
  }
  return k;
}

static bool d_ok(int D) { return D >= 1 && D <= 32; }

extern "C" int ddn_net_param_table(int arch, int D, ddn_tensor_entry* out, int cap) {
  if (!arch_ok(arch) || !d_ok(D)) return DDN_EINVAL;
  const NetSpec& s = get_spec(arch, D);
  for (int i = 0; i < (int)s.ptab.size() && i < cap && out; ++i) out[i] = s.ptab[i];
  return (int)s.ptab.size();
}
extern "C" int ddn_net_buffer_table(int arch, ddn_tensor_entry* out, int cap) {
  if (!arch_ok(arch)) return DDN_EINVAL;
  const NetSpec& s = get_spec(arch, 3);
  for (int i = 0; i < (int)s.btab.size() && i < cap && out; ++i) out[i] = s.btab[i];
  return (int)s.btab.size();
}
extern "C" int64_t ddn_net_param_count(int arch, int D) { return (!arch_ok(arch) || !d_ok(D)) ? DDN_EINVAL : get_spec(arch, D).n_params; }
extern "C" int64_t ddn_net_buffer_count(int arch) { return arch_ok(arch) ? get_spec(arch, 3).n_buffers : DDN_EINVAL; }
extern "C" size_t ddn_net_weight_cache_bytes(int arch, int D) {
  if (!arch_ok(arch) || !d_ok(D)) return 0;
  return (size_t)get_spec(arch, D).n_params * 2 * 2 * sizeof(__nv_bfloat16) + 4096;
}
extern "C" size_t ddn_net_workspace_bytes(int arch, int B, int H, int W, int D, int mode, int precision) {
  return ddn_net_workspace_bytes_v2(arch, B, H, W, D, mode, precision, 0);
}
extern "C" size_t ddn_net_workspace_bytes_v2(int arch, int B, int H, int W, int D, int mode, int precision, int flags) {
  Plan p;
  if (make_plan(&p, arch, B, H, W, D, mode, precision, flags) != 0) return 0;
  return p.total;
}

static int check_ws(const Plan& p, void* ws, size_t bytes) {
  DDN_CHECK_ARG(ws && (reinterpret_cast<uintptr_t>(ws) & 255) == 0, "workspace must be non-null and 256-byte aligned");
  if (bytes < p.total) { set_error("workspace too small: %zu < %zu", bytes, p.total); return DDN_EWORKSPACE; }
  return 0;
}
static int check_groups(int B, int G) {
  DDN_CHECK_ARG(G >= 1 && G <= BN_MAX_GROUPS && B % G == 0, "bn_groups must be 1 or %d and divide the batch (got %d for B=%d)", BN_MAX_GROUPS, G, B);
  return 0;
}

extern "C" int ddn_net_forward(int arch, const float* x, const float* params, float* buffers, float* y,
                               void* workspace, size_t workspace_bytes, int B, int H, int W, int D,
                               int mode, int bn_groups, float momentum, float eps, int precision, float* low_nhwc_out,
                               void* stream) {
  return ddn_net_forward_v2(arch, x, params, buffers, y, workspace, workspace_bytes, B, H, W, D, mode, bn_groups, momentum, eps, precision,
                            low_nhwc_out, 0, stream);
}
extern "C" int ddn_net_forward_v2(int arch, const float* x, const float* params, float* buffers, float* y,
                                  void* workspace, size_t workspace_bytes, int B, int H, int W, int D,
                                  int mode, int bn_groups, float momentum, float eps, int precision, float* low_nhwc_out,
                                  int flags, void* stream) {
  DDN_CHECK_ARG(x && params && buffers && y, "null tensor");
  DDN_TRY(check_groups(B, bn_groups));
  Plan p;
  DDN_TRY(make_plan(&p, arch, B, H, W, D, mode, precision, flags));
  DDN_TRY(check_ws(p, workspace, workspace_bytes));
  Ctx c = {&get_spec(arch, D), &p, (char*)workspace, params, buffers, nullptr, (cudaStream_t)stream, momentum, eps, mode, bn_groups};
  return net_forward(c, x, y, low_nhwc_out);
}

extern "C" int ddn_net_backward(int arch, const float* dy, const float* dlow_nhwc, const float* params, float* grads,
                                void* workspace, size_t workspace_bytes, int B, int H, int W, int D,
                                int mode, int bn_groups, float eps, int precision,
                                ddn_grad_bucket_fn on_bucket, void* user, void* stream) {
  return ddn_net_backward_v2(arch, dy, dlow_nhwc, params, grads, workspace, workspace_bytes, B, H, W, D, mode, bn_groups, eps, precision,
                             0, on_bucket, user, stream);
}
extern "C" int ddn_net_backward_v2(int arch, const float* dy, const float* dlow_nhwc, const float* params, float* grads,
                                   void* workspace, size_t workspace_bytes, int B, int H, int W, int D,
                                   int mode, int bn_groups, float eps, int precision, int flags,
                                   ddn_grad_bucket_fn on_bucket, void* user, void* stream) {
  DDN_CHECK_ARG((dy || dlow_nhwc) && params && grads, "null tensor");
  DDN_CHECK_ARG(mode == DDN_MODE_TRAIN || mode == DDN_MODE_EVAL_SAVE, "backward needs a forward that kept its activations (mode %d)", mode);
  DDN_TRY(check_groups(B, bn_groups));
  Plan p;
  DDN_TRY(make_plan(&p, arch, B, H, W, D, mode, precision, flags));
  DDN_TRY(check_ws(p, workspace, workspace_bytes));
  Ctx c = {&get_spec(arch, D), &p, (char*)workspace, params, nullptr, grads, (cudaStream_t)stream, 0.f, eps, mode, bn_groups};
  return net_backward(c, dy, dlow_nhwc, on_bucket, user);
}

// layer4 + fc, layer3, layer2, then layer1 + stem (net_backward's close_bucket calls)
extern "C" int ddn_net_grad_buckets(int arch, int D, int64_t* offsets, int cap) {
  if (!arch_ok(arch) || !d_ok(D)) return DDN_EINVAL;
  const NetSpec& s = get_spec(arch, D);
  const int64_t b[5] = {s.blocks[s.layer_first[3]].c[0].w_off, s.blocks[s.layer_first[2]].c[0].w_off, s.blocks[s.layer_first[1]].c[0].w_off,
                        0, s.n_params};
  for (int i = 0; i < 5 && i < cap && offsets; ++i) offsets[i] = b[i];
  return 4;
}

// ---- Resnet34_8s names of the entry points above
extern "C" int ddn_resnet34_8s_param_table(int D, ddn_tensor_entry* out, int cap) { return ddn_net_param_table(DDN_ARCH_RESNET34_8S, D, out, cap); }
extern "C" int ddn_resnet34_8s_buffer_table(ddn_tensor_entry* out, int cap) { return ddn_net_buffer_table(DDN_ARCH_RESNET34_8S, out, cap); }
extern "C" int64_t ddn_resnet34_8s_param_count(int D) { return ddn_net_param_count(DDN_ARCH_RESNET34_8S, D); }
extern "C" int64_t ddn_resnet34_8s_buffer_count(void) { return ddn_net_buffer_count(DDN_ARCH_RESNET34_8S); }
extern "C" size_t ddn_resnet34_8s_weight_cache_bytes(int D) { return ddn_net_weight_cache_bytes(DDN_ARCH_RESNET34_8S, D); }
extern "C" size_t ddn_resnet34_8s_workspace_bytes(int B, int H, int W, int D, int mode, int precision) {
  return ddn_net_workspace_bytes(DDN_ARCH_RESNET34_8S, B, H, W, D, mode, precision);
}
extern "C" int ddn_resnet34_8s_forward(const float* x, const float* params, float* buffers, float* y,
                                       void* workspace, size_t workspace_bytes, int B, int H, int W, int D,
                                       int mode, int bn_groups, float momentum, float eps, int precision, float* low_nhwc_out,
                                       void* stream) {
  return ddn_net_forward(DDN_ARCH_RESNET34_8S, x, params, buffers, y, workspace, workspace_bytes, B, H, W, D, mode, bn_groups, momentum, eps,
                         precision, low_nhwc_out, stream);
}
extern "C" int ddn_resnet34_8s_backward(const float* dy, const float* dlow_nhwc, const float* params, float* grads,
                                        void* workspace, size_t workspace_bytes, int B, int H, int W, int D,
                                        int mode, int bn_groups, float eps, int precision,
                                        ddn_grad_bucket_fn on_bucket, void* user, void* stream) {
  return ddn_net_backward(DDN_ARCH_RESNET34_8S, dy, dlow_nhwc, params, grads, workspace, workspace_bytes, B, H, W, D, mode, bn_groups, eps,
                          precision, on_bucket, user, stream);
}
extern "C" int ddn_resnet34_8s_grad_buckets(int D, int64_t* offsets, int cap) { return ddn_net_grad_buckets(DDN_ARCH_RESNET34_8S, D, offsets, cap); }

extern "C" int ddn_resnet34_8s_set_weight_cache(void* cache, size_t bytes, const float* params, uint64_t version, int precision) {
  std::lock_guard<std::mutex> lk(g_wcache_mu);
  WeightCache* wc = nullptr;
  for (auto& w : g_wcaches) if (w.params == params) wc = &w;
  if (!wc) {
    if (!cache) return 0;
    for (auto& w : g_wcaches) if (!w.base) wc = &w;          // reuse a retired slot
    if (!wc) {
      if (g_wcaches.size() >= 64) g_wcaches.erase(g_wcaches.begin());
      g_wcaches.emplace_back();
      wc = &g_wcaches.back();
    }
    wc->params = params; wc->base = nullptr;
  }
  const bool same = wc->base == (char*)cache && wc->bytes == bytes && wc->version == version && wc->precision == precision;
  if (!same) {
    wc->base = (char*)cache; wc->bytes = bytes; wc->version = version; wc->precision = precision;
    wc->fresh = true;           // first use re-packs unconditionally and (re)initialises the device-side fingerprints
  }
  if (!cache) wc->params = nullptr;
  return 0;
}

// ------------------------------------------------------------------------------------------------ single operators
static int conv_out(int in, int k, int stride, int pad, int dil) { return (in + 2 * pad - dil * (k - 1) - 1) / stride + 1; }

extern "C" size_t ddn_conv2d_workspace_bytes(int N, int H, int W, int Cin, int Cout, int k, int stride, int pad, int dil, int precision) {
  size_t wb = align_up(sizeof(float) * (size_t)k * k * Cin * Cout, 256);
  size_t tc = precision == DDN_PRECISION_FP32_SIMT ? 0 : tc_workspace_bytes((size_t)N * H * W * (Cin > Cout ? Cin : Cout));
  return 3 * wb + align_up(tc, 256) + 256;
}

extern "C" int ddn_conv2d_forward(const float* x, const float* w, float* y, int N, int H, int W, int Cin, int Cout,
                                  int k, int stride, int pad, int dil, int precision, void* workspace, size_t workspace_bytes,
                                  void* stream) {
  DDN_CHECK_ARG(x && w && y && workspace, "null tensor");
  DDN_CHECK_ARG(workspace_bytes >= ddn_conv2d_workspace_bytes(N, H, W, Cin, Cout, k, stride, pad, dil, precision), "workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  size_t wb = align_up(sizeof(float) * (size_t)k * k * Cin * Cout, 256);
  int Ho = conv_out(H, k, stride, pad, dil), Wo = conv_out(W, k, stride, pad, dil);
  if (precision != DDN_PRECISION_FP32_SIMT) {
    DDN_CHECK_ARG(tc_conv_supported(Cin, Cout, k, stride, pad, dil, H, W), "shape not supported by the tensor-core path");
    return tc_conv_forward(x, w, y, N, H, W, Cin, Cout, k, stride, pad, dil, precision, (char*)workspace + 3 * wb,
                           workspace_bytes - 3 * wb, st);
  }
  ConvGeom g;
  DDN_TRY(conv_geom_init(&g, N, H, W, Cin, Ho, Wo, Cout, k, k, stride, 1, pad, dil));
  float* wp = (float*)workspace;
  DDN_TRY(launch_pack_weights(w, wp, Cout, Cin, Cin, k, k, 0, st));
  return launch_conv_gather_f32(x, wp, nullptr, y, g, st);
}

extern "C" int ddn_conv2d_backward(const float* x, const float* w, const float* dy, float* dx, float* dw,
                                   int N, int H, int W, int Cin, int Cout, int k, int stride, int pad, int dil,
                                   int precision, void* workspace, size_t workspace_bytes, void* stream) {
  DDN_CHECK_ARG(x && w && dy && dw && workspace, "null tensor");
  DDN_CHECK_ARG(workspace_bytes >= ddn_conv2d_workspace_bytes(N, H, W, Cin, Cout, k, stride, pad, dil, precision), "workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  size_t wb = align_up(sizeof(float) * (size_t)k * k * Cin * Cout, 256);
  int Ho = conv_out(H, k, stride, pad, dil), Wo = conv_out(W, k, stride, pad, dil);
  float* wp = (float*)workspace; float* dwp = (float*)((char*)workspace + wb);
  if (precision != DDN_PRECISION_FP32_SIMT) {
    DDN_CHECK_ARG(tc_conv_supported(Cin, Cout, k, stride, pad, dil, H, W), "shape not supported by the tensor-core path");
    // [wb, 3 wb) holds the fp64 weight-gradient accumulator
    return tc_conv_backward(x, w, dy, dx, nullptr, dw, N, H, W, Cin, Cout, k, stride, pad, dil, precision,
                            (char*)workspace + 3 * wb, workspace_bytes - 3 * wb, reinterpret_cast<double*>(dwp), st);
  }
  ConvGeom g;
  DDN_TRY(conv_geom_init(&g, N, H, W, Cin, Ho, Wo, Cout, k, k, stride, 1, pad, dil));
  DDN_TRY(launch_fill_zero(dwp, sizeof(float) * (size_t)k * k * Cin * Cout, st));
  DDN_TRY(launch_conv_wgrad_f32(x, dy, dwp, g, st));
  DDN_TRY(launch_unpack_wgrad(dwp, dw, Cout, Cin, Cin, k, k, st));
  if (dx) {
    ConvGeom gd;
    DDN_TRY(conv_geom_init(&gd, N, Ho, Wo, Cout, H, W, Cin, k, k, 1, stride, dil * (k - 1) - pad, dil));
    DDN_TRY(launch_pack_weights(w, wp, Cout, Cin, Cin, k, k, 1, st));
    DDN_TRY(launch_conv_gather_f32(dy, wp, nullptr, dx, gd, st));
  }
  return 0;
}

extern "C" size_t ddn_batchnorm_workspace_bytes(int64_t M, int C) {
  (void)M;
  if (!bn_c_supported(C)) return 0;
  return bn_accum_bytes(C) + sizeof(float) * 2 * BN_MAX_GROUPS * C + 256;
}

extern "C" int ddn_batchnorm_forward(const float* x, const float* gamma, const float* beta, const float* residual,
                                     float* y, float* save_mean, float* save_invstd, float* running_mean, float* running_var,
                                     int64_t M, int C, int relu, int training, float momentum, float eps,
                                     void* workspace, size_t workspace_bytes, void* stream) {
  DDN_CHECK_ARG(x && gamma && beta && y && save_mean && save_invstd && workspace, "null tensor");
  DDN_CHECK_ARG(workspace_bytes >= ddn_batchnorm_workspace_bytes(M, C) && ddn_batchnorm_workspace_bytes(M, C) > 0, "bad C or workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  if (training) {
    DDN_CUDA(cudaMemsetAsync(workspace, 0, bn_accum_bytes(C), st));
    DDN_TRY(launch_bn_stats(x, M, C, 1, bn_accum_at(workspace, C), save_mean, save_invstd, running_mean, running_var, momentum, eps, st));
  } else {
    DDN_CHECK_ARG(running_mean && running_var, "eval mode needs running statistics");
    DDN_TRY(launch_bn_eval_stats(running_mean, running_var, C, 1, eps, save_mean, save_invstd, st));
  }
  BnApplyArgs a;
  memset(&a, 0, sizeof(a));
  a.x = x; a.mean = save_mean; a.invstd = save_invstd; a.gamma = gamma; a.beta = beta; a.r = residual; a.y = y;
  a.M = M; a.C = C; a.relu = relu; a.G = 1;
  return launch_bn_apply(a, st);
}

extern "C" int ddn_batchnorm_backward(const float* dy, const float* x, const float* y, const float* gamma,
                                      const float* save_mean, const float* save_invstd, float* dx, float* dgamma, float* dbeta,
                                      float* d_residual, int64_t M, int C, int relu, void* workspace, size_t workspace_bytes, void* stream) {
  DDN_CHECK_ARG(dy && x && gamma && save_mean && save_invstd && dx && dgamma && dbeta && workspace, "null tensor");
  DDN_CHECK_ARG(!relu || y, "relu backward needs the forward output");
  DDN_CHECK_ARG(workspace_bytes >= ddn_batchnorm_workspace_bytes(M, C) && ddn_batchnorm_workspace_bytes(M, C) > 0, "bad C or workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  DDN_CUDA(cudaMemsetAsync(workspace, 0, bn_accum_bytes(C), st));
  BnBwdArgs a;
  memset(&a, 0, sizeof(a));
  a.dy = dy; a.x = x; a.mean = save_mean; a.invstd = save_invstd; a.gamma = gamma; a.y = y;
  a.dx = dx; a.g_out = d_residual; a.dgamma = dgamma; a.dbeta = dbeta;
  a.acc = bn_accum_at(workspace, C); a.sums = reinterpret_cast<float*>((char*)workspace + bn_accum_bytes(C));
  a.M = M; a.C = C; a.relu = relu; a.training = 1; a.G = 1;
  return launch_bn_backward(a, st);
}

// ---- tensor-core convolutions with their fused epilogues (the variants the network's forward and backward run)
// workspace: [BatchNorm accumulator + ticket][fold scale | shift][tensor-core staging (stage_planes)]
static bool is_stem_shape(int Cin, int Cout, int k, int stride, int pad, int dil) {
  return Cin == 3 && Cout == 64 && k == 7 && stride == 2 && pad == 3 && dil == 1;
}
static size_t fused_head_bytes(int C) { return bn_accum_bytes(C) + align_up(sizeof(float) * 2 * (size_t)C, 256); }

extern "C" size_t ddn_conv2d_fused_workspace_bytes(int N, int H, int W, int Cin, int Cout, int k, int stride, int pad, int dil,
                                                   int precision) {
  if (N < 1 || H < 1 || W < 1 || Cin < 1 || Cout < 1 || precision == DDN_PRECISION_FP32_SIMT) return 0;
  const int C = Cin > Cout ? Cin : Cout;
  size_t act = (size_t)N * H * W * C;      // the stem stages its 7x7/2 patches instead of the NCHW input
  if (is_stem_shape(Cin, Cout, k, stride, pad, dil)) act = (size_t)N * conv_out(H, 7, 2, 3, 1) * conv_out(W, 7, 2, 3, 1) * 192;
  return fused_head_bytes(C) + tc_workspace_bytes(act) + 1024;
}

// every check of the fused entries, before anything is launched
static int check_fused(int N, int H, int W, int Cin, int Cout, int k, int stride, int pad, int dil, int G, int precision,
                       size_t ws_bytes, bool allow_stem) {
  DDN_CHECK_ARG(precision >= DDN_PRECISION_FP32_SIMT && precision <= DDN_PRECISION_BF16, "unknown precision %d", precision);
  if (precision == DDN_PRECISION_FP32_SIMT) {
    set_error("the fused conv epilogues exist on the tensor-core path only (precision %d)", precision);
    return DDN_EUNSUPPORTED;
  }
  DDN_CHECK_ARG(N >= 1 && H >= 8 && W >= 8, "bad sizes N=%d H=%d W=%d", N, H, W);
  DDN_CHECK_ARG(G >= 1 && G <= BN_MAX_GROUPS && N % G == 0, "bn_groups must be 1 or %d and divide N (got %d for N=%d)", BN_MAX_GROUPS, G, N);
  const bool stem = is_stem_shape(Cin, Cout, k, stride, pad, dil);
  if (stem) {
    if (!allow_stem) { set_error("the stem patch GEMM has no fused variant here"); return DDN_EUNSUPPORTED; }
  } else if (!tc_conv_supported(Cin, Cout, k, stride, pad, dil, H, W)) {
    set_error("shape not supported by the tensor-core path (Cin=%d Cout=%d k=%d stride=%d pad=%d dil=%d H=%d W=%d)", Cin, Cout, k, stride,
              pad, dil, H, W);
    return DDN_EUNSUPPORTED;
  }
  DDN_CHECK_ARG(ws_bytes >= ddn_conv2d_fused_workspace_bytes(N, H, W, Cin, Cout, k, stride, pad, dil, precision), "workspace too small");
  return 0;
}

extern "C" int ddn_conv2d_bn_stats_forward(const float* x, const float* w, float* raw, float* mean, float* invstd, float* running_mean,
                                           float* running_var, int N, int H, int W, int Cin, int Cout, int k, int stride, int pad,
                                           int dil, int bn_groups, float momentum, float eps, int precision, void* workspace,
                                           size_t workspace_bytes, void* stream) {
  DDN_CHECK_ARG(x && w && raw && mean && invstd && workspace, "null tensor");
  DDN_CHECK_ARG(!running_mean == !running_var, "running_mean and running_var go together");
  DDN_TRY(check_fused(N, H, W, Cin, Cout, k, stride, pad, dil, bn_groups, precision, workspace_bytes, true));
  cudaStream_t st = (cudaStream_t)stream;
  const int Ho = conv_out(H, k, stride, pad, dil), Wo = conv_out(W, k, stride, pad, dil);
  const int C = Cin > Cout ? Cin : Cout;
  char* ws = (char*)workspace;
  BnFwdFinal fin;
  fin.a = bn_accum_at(ws, C);
  fin.mean = mean; fin.invstd = invstd; fin.running_mean = running_mean; fin.running_var = running_var;
  fin.count = (int64_t)N / bn_groups * Ho * Wo; fin.G = bn_groups; fin.C = Cout; fin.momentum = momentum; fin.eps = eps;
  DDN_CUDA(cudaMemsetAsync(ws, 0, bn_accum_bytes(C), st));
  char* stage = ws + fused_head_bytes(C);
  const size_t stage_bytes = workspace_bytes - fused_head_bytes(C);
  void* wws; TcPlanes px, pdy, pup;
  if (is_stem_shape(Cin, Cout, k, stride, pad, dil)) {      // x is NCHW [N,3,H,W]: 7x7/2 patch planes, then the K = 192 GEMM
    DDN_TRY(stage_planes(stage, stage_bytes, (size_t)N * Ho * Wo * 192, 0, 0, &wws, &px, &pdy, &pup));
    DDN_TRY(tc_stem_patches(x, const_cast<__nv_bfloat16*>(px.hi), const_cast<__nv_bfloat16*>(px.lo), N, H, W, precision, st));
    return tc_stem_forward(px, w, nullptr, raw, &fin, N, Ho, Wo, precision, wws, tc_weight_ws_bytes(), st);
  }
  DDN_TRY(stage_planes(stage, stage_bytes, (size_t)N * H * W * Cin, 0, 0, &wws, &px, &pdy, &pup));
  DDN_TRY(tc_split(x, const_cast<__nv_bfloat16*>(px.hi), const_cast<__nv_bfloat16*>(px.lo), (int64_t)N * H * W * Cin, precision, st));
  return tc_conv_planes(px, w, nullptr, raw, nullptr, &fin, N, H, W, Cin, Cout, k, stride, dil, 0, precision, wws, tc_weight_ws_bytes(), st);
}

extern "C" int ddn_conv2d_folded_forward(const float* x, const float* w, const float* gamma, const float* beta, const float* running_mean,
                                         const float* running_var, const float* addend, float* y, void* y_hi, void* y_lo,
                                         int N, int H, int W, int Cin, int Cout, int k, int stride, int pad, int dil, int relu, float eps,
                                         int precision, void* workspace, size_t workspace_bytes, void* stream) {
  DDN_CHECK_ARG(x && w && gamma && beta && running_mean && running_var && workspace, "null tensor");
  DDN_CHECK_ARG(y || y_hi, "the folded epilogue needs an output: y and / or the y_hi plane");
  DDN_CHECK_ARG(y_hi || !y_lo, "y_lo is the low plane of y_hi");
  DDN_TRY(check_fused(N, H, W, Cin, Cout, k, stride, pad, dil, 1, precision, workspace_bytes, false));
  cudaStream_t st = (cudaStream_t)stream;
  const int C = Cin > Cout ? Cin : Cout;
  char* ws = (char*)workspace;
  float* scale = reinterpret_cast<float*>(ws + bn_accum_bytes(C)); float* shift = scale + Cout;
  char* stage = ws + fused_head_bytes(C);
  void* wws; TcPlanes px, pdy, pup;
  DDN_TRY(stage_planes(stage, workspace_bytes - fused_head_bytes(C), (size_t)N * H * W * Cin, 0, 0, &wws, &px, &pdy, &pup));
  DDN_TRY(launch_bn_fold(running_mean, running_var, gamma, beta, Cout, eps, scale, shift, st));
  DDN_TRY(tc_split(x, const_cast<__nv_bfloat16*>(px.hi), const_cast<__nv_bfloat16*>(px.lo), (int64_t)N * H * W * Cin, precision, st));
  TcFoldedEpilogue ep = {scale, shift, relu ? 1 : 0, (__nv_bfloat16*)y_hi, (__nv_bfloat16*)y_lo};
  return tc_conv_planes(px, w, nullptr, y, addend, nullptr, N, H, W, Cin, Cout, k, stride, dil, 0, precision, wws, tc_weight_ws_bytes(), st,
                        &ep);
}

extern "C" int ddn_conv2d_backward_data_bn_stats(const float* w, const float* dy, const float* addend, const float* raw, const float* mean,
                                                 const float* invstd, const float* gamma, const float* beta, const void* y_hi,
                                                 float* dx, float* dgamma, float* dbeta, float* sums,
                                                 int N, int H, int W, int Cin, int Cout, int k, int stride, int pad, int dil,
                                                 int bn_groups, int precision, void* workspace, size_t workspace_bytes, void* stream) {
  DDN_CHECK_ARG(w && dy && raw && mean && invstd && dx && dgamma && dbeta && sums && workspace, "null tensor");
  DDN_CHECK_ARG(y_hi || (gamma && beta), "the recomputed ReLU mask (y_hi == NULL) needs gamma and beta");
  DDN_TRY(check_fused(N, H, W, Cin, Cout, k, stride, pad, dil, bn_groups, precision, workspace_bytes, false));
  cudaStream_t st = (cudaStream_t)stream;
  const int Ho = conv_out(H, k, stride, pad, dil), Wo = conv_out(W, k, stride, pad, dil);
  const int C = Cin > Cout ? Cin : Cout;
  char* ws = (char*)workspace;
  TcBwdStats bst;
  memset(&bst, 0, sizeof(bst));
  bst.raw = raw; bst.y_hi = (const __nv_bfloat16*)y_hi; bst.mean = mean; bst.invstd = invstd; bst.gamma = gamma; bst.beta = beta;
  bst.relu = 1;
  bst.fin.a = bn_accum_at(ws, C); bst.fin.sums = sums; bst.fin.dgamma = dgamma; bst.fin.dbeta = dbeta; bst.fin.G = bn_groups; bst.fin.C = Cin;
  char* stage = ws + fused_head_bytes(C);
  void* wws; TcPlanes px, pdy, pup;
  DDN_TRY(stage_planes(stage, workspace_bytes - fused_head_bytes(C), 0, (size_t)N * Ho * Wo * Cout, stride == 2 ? (size_t)N * H * W * Cout : 0,
                       &wws, &px, &pdy, &pup));
  DDN_CUDA(cudaMemsetAsync(ws, 0, bn_accum_bytes(C), st));
  if (stride == 2)      // zero insertion into the `up` planes, then a stride-1 data gradient
    return tc_dgrad_strided(dy, pup, w, nullptr, dx, addend, N, H, W, Cin, Cout, k, precision, wws, tc_weight_ws_bytes(), st, &bst);
  DDN_TRY(tc_split(dy, const_cast<__nv_bfloat16*>(pdy.hi), const_cast<__nv_bfloat16*>(pdy.lo), (int64_t)N * Ho * Wo * Cout, precision, st));
  return tc_conv_planes(pdy, w, nullptr, dx, addend, nullptr, N, H, W, Cin, Cout, k, 1, dil, 1, precision, wws, tc_weight_ws_bytes(), st,
                        nullptr, &bst);
}

// ---- the stem alone: the pool forward the network runs after conv1 + bn1 statistics, and the network's stem backward
extern "C" int ddn_stem_pool_forward(const float* raw, const float* mean, const float* invstd, const float* gamma, const float* beta,
                                     float* y, void* y_hi, void* y_lo, void* argmax, int N, int Hc, int Wc, int G, void* stream) {
  DDN_CHECK_ARG(raw && mean && invstd && gamma && beta && argmax, "null tensor");
  DDN_CHECK_ARG(y || y_hi, "the pool needs an output: y and / or the y_hi plane");
  DDN_CHECK_ARG(y_hi || !y_lo, "y_lo is the low plane of y_hi");
  DDN_CHECK_ARG(N >= 1 && Hc >= 1 && Wc >= 1, "bad sizes N=%d Hc=%d Wc=%d", N, Hc, Wc);
  DDN_TRY(check_groups(N, G));
  return launch_stem_bn_relu_pool(raw, mean, invstd, gamma, beta, y, reinterpret_cast<uint8_t*>(argmax), (__nv_bfloat16*)y_hi,
                                  (__nv_bfloat16*)y_lo, N, Hc, Wc, 64, G, (cudaStream_t)stream);
}

// workspace of ddn_stem_backward: byte offsets, 256-byte aligned
struct StemWs { size_t acc, sums, g, dx, patch_hi, patch_lo, dx_hi, dx_lo, dwp, x4, dwp_f32, total; };
static bool stem_ws_plan(int N, int H, int W, int precision, StemWs* w) {
  if (N < 1 || H < 1 || W < 1 || precision < DDN_PRECISION_FP32_SIMT || precision > DDN_PRECISION_BF16) return false;
  memset(w, 0, sizeof(*w));
  size_t cur = 0;
  auto alloc = [&](size_t bytes) { size_t o = cur; cur += align_up(bytes, 256); return o; };
  const size_t m1 = (size_t)N * conv_out(H, 7, 2, 3, 1) * conv_out(W, 7, 2, 3, 1);
  w->acc = alloc(bn_accum_bytes(64));
  w->sums = alloc(sizeof(float) * 2 * BN_MAX_GROUPS * 64);
  w->g = alloc(sizeof(float) * m1 * 64);
  w->dx = alloc(sizeof(float) * m1 * 64);
  if (precision != DDN_PRECISION_FP32_SIMT) {
    w->patch_hi = alloc(2 * m1 * 192); w->patch_lo = alloc(2 * m1 * 192);
    w->dx_hi = alloc(2 * m1 * 64); w->dx_lo = alloc(2 * m1 * 64);
    w->dwp = alloc(sizeof(double) * 64 * 192);
  } else {
    w->x4 = alloc(sizeof(float) * (size_t)N * H * W * 4);
    w->dwp_f32 = alloc(sizeof(float) * 7 * 7 * 4 * 64);
  }
  w->total = cur;
  return true;
}

extern "C" size_t ddn_stem_workspace_bytes(int N, int H, int W, int precision) {
  StemWs w;
  return stem_ws_plan(N, H, W, precision, &w) ? w.total : 0;
}

extern "C" int ddn_stem_backward(const float* x_nchw, const float* raw, const float* mean, const float* invstd, const float* gamma,
                                 const float* beta, const void* argmax, const float* dy_pool, float* g_out, float* dx_bn,
                                 void* dx_hi, void* dx_lo, float* dgamma, float* dbeta, float* dw_conv1, int N, int H, int W, int G,
                                 int training, int precision, void* workspace, size_t workspace_bytes, void* stream) {
  DDN_CHECK_ARG(x_nchw && raw && mean && invstd && gamma && beta && argmax && dy_pool && dgamma && dbeta && dw_conv1, "null tensor");
  DDN_CHECK_ARG(precision >= DDN_PRECISION_FP32_SIMT && precision <= DDN_PRECISION_BF16, "unknown precision %d", precision);
  DDN_CHECK_ARG(N >= 1 && H >= 1 && W >= 1, "bad sizes N=%d H=%d W=%d", N, H, W);
  DDN_TRY(check_groups(N, G));
  const int H1 = conv_out(H, 7, 2, 3, 1), W1 = conv_out(W, 7, 2, 3, 1);
  DDN_CHECK_ARG(N <= 65535 && H1 <= 65535, "stem: batch / height too large for the launch grid");
  StemWs w;
  stem_ws_plan(N, H, W, precision, &w);
  DDN_CHECK_ARG(workspace && (reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "workspace must be non-null and 256-byte aligned");
  if (workspace_bytes < w.total) { set_error("workspace too small: %zu < %zu", workspace_bytes, w.total); return DDN_EWORKSPACE; }
  cudaStream_t st = (cudaStream_t)stream;
  char* ws = (char*)workspace;
  auto bf = [&](size_t off) { return reinterpret_cast<__nv_bfloat16*>(ws + off); };
  DDN_CUDA(cudaMemsetAsync(ws + w.acc, 0, bn_accum_bytes(64), st));
  StemBwdArgs a;
  memset(&a, 0, sizeof(a));
  a.dy_pool = dy_pool; a.argmax = reinterpret_cast<const uint8_t*>(argmax); a.raw = raw; a.mean = mean; a.invstd = invstd;
  a.gamma = gamma; a.beta = beta; a.dgamma = dgamma; a.dbeta = dbeta;
  a.g = g_out ? g_out : reinterpret_cast<float*>(ws + w.g);
  a.acc = bn_accum_at(ws + w.acc, 64); a.sums = reinterpret_cast<float*>(ws + w.sums);
  a.N = N; a.H = H; a.W = W; a.H1 = H1; a.W1 = W1; a.G = G; a.training = training ? 1 : 0; a.precision = precision;
  if (precision == DDN_PRECISION_FP32_SIMT) {
    a.x4 = reinterpret_cast<float*>(ws + w.x4); a.dwp_f32 = reinterpret_cast<float*>(ws + w.dwp_f32); a.dw = dw_conv1;
    a.dx = dx_bn ? dx_bn : reinterpret_cast<float*>(ws + w.dx);
    DDN_TRY(launch_nchw_to_nhwc4(x_nchw, const_cast<float*>(a.x4), N, H, W, st));
    return stem_backward(a, st);
  }
  a.patches = TcPlanes{bf(w.patch_hi), bf(w.patch_lo)};
  a.dx_hi = dx_hi ? (__nv_bfloat16*)dx_hi : bf(w.dx_hi); a.dx_lo = dx_lo ? (__nv_bfloat16*)dx_lo : bf(w.dx_lo);
  a.dx = dx_bn; a.dwp = reinterpret_cast<double*>(ws + w.dwp);
  DDN_CUDA(cudaMemsetAsync(a.dwp, 0, sizeof(double) * 64 * 192, st));
  DDN_TRY(tc_stem_patches(x_nchw, bf(w.patch_hi), bf(w.patch_lo), N, H, W, precision, st));
  DDN_TRY(stem_backward(a, st));
  const TcUnpackEntry e = stem_unpack_entry(0, 0);
  return tc_unpack_wgrads(&e, 1, a.dwp, dw_conv1, st);
}
