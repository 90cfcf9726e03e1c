// Conv-graph runtime behind seam S1 (`self.model(image)`, simple_romp/romp/main.py:112).
//
// The host layer (romp_b200/graph.py) walks the reference's state-dict layout
// (HigherResolutionNet model.py:246-417, ROMPv1 head :420-481), folds BatchNorm and emits one fused
// conv op per Conv2d.  This file owns: tensor table, liveness-based buffer planning for the NHWC
// activation workspace, weight packing/upload per engine, launch sequencing and CUDA-graph replay.
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <array>
#include <map>
#include <mutex>
#include <vector>

#include "common.cuh"
#include "conv_tc.cuh"

namespace b200romp {

static thread_local std::string g_last_error;

void set_error(const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_last_error = buf;
}

void* upload(const void* host, size_t bytes, std::vector<void*>* allocs) {
  void* d = nullptr;
  cudaError_t e = cudaMalloc(&d, bytes);
  if (e == cudaSuccess) {
    allocs->push_back(d);
    e = cudaMemcpy(d, host, bytes, cudaMemcpyHostToDevice);
  }
  if (e != cudaSuccess) {
    set_error("upload of %zu bytes failed: %s", bytes, cudaGetErrorString(e));
    return nullptr;
  }
  return d;
}

struct Tensor {
  int H, W, C, dtype, nchw, external;
  void* ptr = nullptr;        // device pointer (workspace slice or bound external / constant)
  bool constant = false;
  int first_def = -1, last_use = -1;
  size_t frame_bytes() const { return (size_t)H * W * C * dtype_size(dtype); }
};

// The kernel that runs an op.  Sum and MaxPool are set when the op is added, WgmmaBlock and WgmmaBottleneck by
// fuse_chains; every other conv is Simt until choose_kernel decides at finalize.  Generic7x7 and Deconv4x4 are the
// CUDA-core kernels of resnet_ops.cu; a Wgmma or WgmmaBlock plan with tc.fold runs on the pixel-pair view
// (fold_pixel_pairs).
enum class Kernel { Sum, MaxPool, Simt, Generic7x7, Deconv4x4, Wgmma, WgmmaStem, WgmmaConv1d, WgmmaBlock, WgmmaBottleneck };

// one conv as added: its descriptor, OIHW fp32 weights and [cout] bias (both freed at finalize)
struct Conv {
  b200romp_conv_desc d;
  std::vector<float> w, b;
  // inside a fused op, for every conv but the last: its output is an intermediate that other ops read as well, so the
  // fused kernel writes it and it gets a buffer
  bool stored = false;
};

struct Op {
  Kernel kernel = Kernel::Simt;
  b200romp_sum_desc sum;
  // a conv: the chain of convs the op runs, one for a plain conv and the convs it replaces for a fused one; d is then the
  // chain as one conv (input and residual = the first conv's input, output = the last conv's).  Sum / maxpool: no parts,
  // d.out / d.in mirror out / base or in, d.res = -1.
  b200romp_conv_desc d;
  std::vector<Conv> parts;
  float* d_w_simt = nullptr;           // CUDA-core kernels only: [tap][cin][coutPad]
  float* d_bias = nullptr;             // the last conv's bias, [coutPad]
  int coutPad = 0;
  TcConvPlan tc;                       // wgmma kernels: packed weights, tensor maps, tiling
  int lane = 0;                        // concurrency lane inside the captured CUDA graph (b200romp_net_set_lane)
};

// the tensors an op writes: its output, and a fused op's stored intermediates
static std::vector<int> op_outputs(const Op& op) {
  std::vector<int> o{op.d.out};
  for (size_t k = 0; k + 1 < op.parts.size(); ++k)
    if (op.parts[k].stored) o.push_back(op.parts[k].d.out);
  return o;
}

static bool on_wgmma(Kernel k) {
  return k == Kernel::Wgmma || k == Kernel::WgmmaStem || k == Kernel::WgmmaConv1d || k == Kernel::WgmmaBlock || k == Kernel::WgmmaBottleneck;
}

}  // namespace b200romp

using namespace b200romp;

struct b200romp_net {
  int device = 0;
  int sm_count = 132;
  bool finalized = false;
  int max_batch = 0;
  std::vector<Tensor> tensors;
  std::vector<Op> ops;
  std::vector<void*> device_allocs;
  char* workspace = nullptr;
  size_t workspace_bytes = 0;
  struct GraphKey {
    int batch;
    std::vector<void*> ext;
    bool operator<(const GraphKey& o) const { return batch != o.batch ? batch < o.batch : ext < o.ext; }
  };
  std::map<GraphKey, cudaGraphExec_t> graphs;
  bool use_graph = true;
  // multi-lane capture: independent ops (the HRNet branches, the three heads) are captured on separate streams so that the
  // ramp-up / tail of one persistent conv kernel overlaps the body of a kernel of another branch
  static constexpr int kLanes = 4;
  cudaStream_t lane_stream[kLanes] = {nullptr, nullptr, nullptr, nullptr};
  std::vector<cudaEvent_t> op_done;     // one event per op, recorded on the op's lane during capture
  cudaEvent_t fork_ev = nullptr;
  bool use_lanes = false;
};

// `allow_unbound` (planning): a tensor without storage yet - internal before buffer planning, external before
// b200romp_net_bind - leaves a null pointer.  Launches require every pointer.
static int fill_params(const b200romp_net* net, const Op& op, int batch, bool allow_unbound, ConvParams* out) {
  const b200romp_conv_desc& d = op.d;
  const Tensor& ti = net->tensors[d.in];
  const Tensor& to = net->tensors[d.out];
  ConvParams p;
  memset(&p, 0, sizeof(p));
  p.in = ti.ptr; p.out = to.ptr;
  p.w = op.d_w_simt; p.bias = op.d_bias;
  p.B = batch;
  p.Hin = ti.H; p.Win = ti.W; p.in_C = ti.C; p.in_c_off = d.in_c_off; p.cin = d.cin;
  conv_out_hw(d.ksize, d.stride, ti.H, ti.W, &p.Hout, &p.Wout);   // 13 = Conv1d 1x3, 42 = ConvTranspose2d(4,2,1)
  p.out_C = to.C; p.out_c_off = d.out_c_off; p.cout = d.cout; p.coutPad = op.coutPad;
  p.up = d.upsample;
  if (d.res >= 0) {
    const Tensor& tr = net->tensors[d.res];
    p.res = tr.ptr; p.res_C = tr.C; p.res_c_off = op.d.res_c_off; p.res_broadcast = d.res_broadcast;
    p.res_dtype = tr.dtype;
  }
  p.relu = d.relu; p.pow_channel = d.pow_channel; p.out_nchw = to.nchw;
  p.in_dtype = ti.dtype; p.out_dtype = to.dtype; p.input_norm = d.input_norm;
  if (op.tc.fold) {   // the same bytes seen as [B, H, W/2, 2C]: two horizontally adjacent pixels form one 64-channel pixel
    p.Win /= 2; p.Wout /= 2;
    p.in_C *= 2; p.cin *= 2; p.out_C *= 2; p.cout *= 2; p.res_C *= 2;
  }
  if (!allow_unbound && (!p.in || !p.out)) {
    set_error("op uses an unbound tensor (in=%d out=%d)", d.in, d.out);
    return B200ROMP_ESTATE;
  }
  *out = p;
  return B200ROMP_OK;
}

// channel slices [a, a + n) and [b, b + m) of one tensor share a channel
static bool slices_overlap(int a, int n, int b, int m) { return a < b + m && b < a + n; }

static int validate_desc(const std::vector<Tensor>& T, const b200romp_conv_desc& d) {
  const int res_c_off = d.res_c_off;
  auto ok_id = [&](int id) { return id >= 0 && id < (int)T.size(); };
  B2R_REQUIRE(ok_id(d.in) && ok_id(d.out) && (d.res == -1 || ok_id(d.res)), "conv: bad tensor id");
  B2R_REQUIRE((d.ksize == 1 || d.ksize == 3 || d.ksize == 7 || (d.ksize == 13 && d.stride == 1 && d.upsample == 1) ||
               (d.ksize == 42 && d.stride == 2 && d.upsample == 1)) && (d.stride == 1 || d.stride == 2),
              "conv: ksize/stride unsupported");
  B2R_REQUIRE(d.upsample == 1 || d.upsample == 2 || d.upsample == 4 || d.upsample == 8, "conv: upsample must be 1,2,4,8");
  const Tensor& ti = T[d.in];
  const Tensor& to = T[d.out];
  B2R_REQUIRE(!ti.nchw, "conv: NCHW inputs unsupported");
  B2R_REQUIRE(d.cin > 0 && d.in_c_off >= 0 && d.in_c_off + d.cin <= ti.C, "conv: input channel slice out of range");
  B2R_REQUIRE(d.cout > 0 && d.out_c_off >= 0 && d.out_c_off + d.cout <= to.C, "conv: output channel slice out of range");
  int Ho, Wo;
  conv_out_hw(d.ksize, d.stride, ti.H, ti.W, &Ho, &Wo);
  B2R_REQUIRE(Ho * d.upsample == to.H && Wo * d.upsample == to.W, "conv: output tensor is %dx%d, op produces %dx%d",
              to.H, to.W, Ho * d.upsample, Wo * d.upsample);
  B2R_REQUIRE(ti.dtype != B200ROMP_U8 || d.input_norm || d.ksize == 7, "conv: u8 input requires input_norm (or the 7x7 stem)");
  B2R_REQUIRE(to.dtype != B200ROMP_U8, "conv: u8 output unsupported");
  B2R_REQUIRE(!to.nchw || to.dtype == B200ROMP_F32, "conv: NCHW output must be fp32");
  if (d.res >= 0) {
    const Tensor& tr = T[d.res];
    B2R_REQUIRE(tr.H == to.H && tr.W == to.W && !tr.nchw && tr.dtype != B200ROMP_U8, "conv: residual shape/dtype mismatch");
    B2R_REQUIRE(res_c_off >= 0 && res_c_off + d.cout <= tr.C, "conv: residual channel slice out of range");
  }
  // Aliasing: other CTAs read the input's halo and all its channels while the output is written, so the input slice must not
  // overlap the output slice of the same tensor; the residual is read elementwise, so it may also be the output slice itself.
  B2R_REQUIRE(d.in != d.out || !slices_overlap(d.in_c_off, d.cin, d.out_c_off, d.cout),
              "conv: input slice [%d, %d) of tensor %d overlaps the output slice [%d, %d)", d.in_c_off, d.in_c_off + d.cin, d.in,
              d.out_c_off, d.out_c_off + d.cout);
  B2R_REQUIRE(d.res != d.out || !slices_overlap(res_c_off, d.cout, d.out_c_off, d.cout) || (res_c_off == d.out_c_off && !d.res_broadcast),
              "conv: residual slice [%d, %d) of tensor %d overlaps the output slice [%d, %d) without being it", res_c_off,
              res_c_off + d.cout, d.res, d.out_c_off, d.out_c_off + d.cout);
  return B200ROMP_OK;
}

extern "C" {

int b200romp_version(void) { return B200ROMP_VERSION; }
const char* b200romp_last_error(void) { return g_last_error.c_str(); }

int b200romp_device_info(int* sm_count, int* cc_major, int* cc_minor) {
  int dev = 0;
  B2R_CUDA_OK(cudaGetDevice(&dev));
  cudaDeviceProp prop;
  B2R_CUDA_OK(cudaGetDeviceProperties(&prop, dev));
  if (sm_count) *sm_count = prop.multiProcessorCount;
  if (cc_major) *cc_major = prop.major;
  if (cc_minor) *cc_minor = prop.minor;
  return B200ROMP_OK;
}

b200romp_net* b200romp_net_create(int device) {
  if (cudaSetDevice(device) != cudaSuccess) {
    set_error("cudaSetDevice(%d) failed - libb200romp needs a CUDA device (no CPU fallback)", device);
    return nullptr;
  }
  b200romp_net* net = new b200romp_net();
  net->device = device;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) net->sm_count = prop.multiProcessorCount;
  const char* ng = getenv("B200ROMP_NO_GRAPH");
  net->use_graph = !(ng && ng[0] == '1');
  const char* nl = getenv("B200ROMP_LANES");       // multi-lane capture is opt-in (see graph.py: concurrent persistent convs share L2)
  net->use_lanes = nl && nl[0] == '1';
  return net;
}

void b200romp_net_destroy(b200romp_net* net) {
  if (!net) return;
  cudaSetDevice(net->device);
  for (auto& kv : net->graphs) cudaGraphExecDestroy(kv.second);
  for (cudaEvent_t e : net->op_done) cudaEventDestroy(e);
  if (net->fork_ev) cudaEventDestroy(net->fork_ev);
  for (int l = 1; l < b200romp_net::kLanes; ++l)
    if (net->lane_stream[l]) cudaStreamDestroy(net->lane_stream[l]);
  for (void* p : net->device_allocs) cudaFree(p);
  if (net->workspace) cudaFree(net->workspace);
  delete net;
}

int b200romp_net_add_tensor(b200romp_net* net, int H, int W, int C, int dtype, int nchw, int external) {
  B2R_REQUIRE(net && !net->finalized, "add_tensor: net is null or finalized");
  B2R_REQUIRE(H > 0 && W > 0 && C > 0 && dtype >= 0 && dtype <= 2, "add_tensor: bad shape/dtype");
  Tensor t;
  t.H = H; t.W = W; t.C = C; t.dtype = dtype; t.nchw = nchw; t.external = external;
  net->tensors.push_back(t);
  return (int)net->tensors.size() - 1;
}

// Constant tensor without a batch dimension (e.g. the coord-conv bias map of the ROMP head).
int b200romp_net_add_const_tensor(b200romp_net* net, int H, int W, int C, int dtype, const void* host_data) {
  int id = b200romp_net_add_tensor(net, H, W, C, dtype, 0, 0);
  if (id < 0) return id;
  Tensor& t = net->tensors[id];
  t.constant = true;
  B2R_CUDA_OK(cudaSetDevice(net->device));
  t.ptr = upload(host_data, t.frame_bytes(), &net->device_allocs);
  return t.ptr ? id : B200ROMP_ECUDA;
}

int b200romp_net_add_conv(b200romp_net* net, const b200romp_conv_desc* desc, const float* weight, const float* bias) {
  B2R_REQUIRE(net && !net->finalized && desc && weight, "add_conv: bad arguments");
  int rc = validate_desc(net->tensors, *desc);
  if (rc) return rc;
  Conv c;
  c.d = *desc;
  c.w.assign(weight, weight + (size_t)desc->cout * desc->cin * conv_taps(desc->ksize));
  c.b.assign(desc->cout, 0.f);
  if (bias) c.b.assign(bias, bias + desc->cout);
  Op op;
  op.d = *desc;
  op.parts.push_back(std::move(c));
  net->ops.push_back(std::move(op));
  return (int)net->ops.size() - 1;
}

int b200romp_net_add_sum(b200romp_net* net, const b200romp_sum_desc* desc) {
  B2R_REQUIRE(net && desc && !net->finalized, "add_sum: bad arguments or net already finalized");
  const auto& T = net->tensors;
  const int nT = (int)T.size();
  B2R_REQUIRE(desc->out >= 0 && desc->out < nT && desc->base >= 0 && desc->base < nT, "add_sum: tensor id out of range");
  B2R_REQUIRE(desc->n_terms >= 1 && desc->n_terms <= 4, "add_sum: n_terms must be 1..4");
  const Tensor& to = T[desc->out];
  const Tensor& tb = T[desc->base];
  B2R_REQUIRE(!to.nchw && !tb.nchw && to.dtype != B200ROMP_U8 && tb.dtype != B200ROMP_U8, "add_sum: NHWC bf16/fp32 tensors only");
  B2R_REQUIRE(to.C % 8 == 0 && tb.H == to.H && tb.W == to.W && tb.C == to.C, "add_sum: base/out shape mismatch (C %% 8 == 0)");
  for (int k = 0; k < desc->n_terms; ++k) {
    B2R_REQUIRE(desc->term[k] >= 0 && desc->term[k] < nT, "add_sum: term tensor id out of range");
    const Tensor& tt = T[desc->term[k]];
    const int u = desc->up[k];
    B2R_REQUIRE(u == 1 || u == 2 || u == 4 || u == 8, "add_sum: up must be 1,2,4,8");
    const int co = desc->term_c_off[k];
    B2R_REQUIRE(!tt.nchw && tt.dtype != B200ROMP_U8 && tt.C % 8 == 0 && co >= 0 && co % 8 == 0 && co + to.C <= tt.C &&
                    tt.H * u == to.H && tt.W * u == to.W,
                "add_sum: term %d is %dx%dx%d (slice from channel %d), expected %dx%dx%d", k, tt.H, tt.W, tt.C, co, to.H / u, to.W / u, to.C);
  }
  // aliasing: a base or term that is the output tensor has its shape, so up 1 and the whole, identical slice (elementwise)
  Op op;
  op.kernel = Kernel::Sum;
  op.sum = *desc;
  memset(&op.d, 0, sizeof(op.d));
  op.d.out = desc->out; op.d.in = desc->base; op.d.res = -1;
  net->ops.push_back(std::move(op));
  return (int)net->ops.size() - 1;
}

int b200romp_net_add_maxpool(b200romp_net* net, int in, int out) {
  B2R_REQUIRE(net && !net->finalized, "add_maxpool: net is null or finalized");
  const int nT = (int)net->tensors.size();
  B2R_REQUIRE(in >= 0 && in < nT && out >= 0 && out < nT, "add_maxpool: tensor id out of range");
  const Tensor& ti = net->tensors[in];
  const Tensor& to = net->tensors[out];
  B2R_REQUIRE(!ti.nchw && !to.nchw && ti.dtype == to.dtype && ti.dtype != B200ROMP_U8 && ti.C == to.C, "add_maxpool: NHWC bf16/fp32 tensors of equal C");
  B2R_REQUIRE(in != out, "add_maxpool: input tensor %d is the output tensor (a window is read while its neighbours are written)", in);
  B2R_REQUIRE(to.H == (ti.H + 2 - 3) / 2 + 1 && to.W == (ti.W + 2 - 3) / 2 + 1, "add_maxpool: output must be %dx%d", (ti.H - 1) / 2 + 1, (ti.W - 1) / 2 + 1);
  Op op;
  op.kernel = Kernel::MaxPool;
  memset(&op.d, 0, sizeof(op.d));
  memset(&op.sum, 0, sizeof(op.sum));
  op.d.in = in; op.d.out = out; op.d.res = -1;
  net->ops.push_back(std::move(op));
  return (int)net->ops.size() - 1;
}

static int fill_sum_params(b200romp_net* net, const Op& op, int batch, SumParams* out) {
  SumParams p;
  memset(&p, 0, sizeof(p));
  const Tensor& to = net->tensors[op.sum.out];
  const Tensor& tb = net->tensors[op.sum.base];
  B2R_REQUIRE(to.ptr && tb.ptr, "sum op: unbound tensor");
  p.base = tb.ptr; p.base_dt = tb.dtype; p.out = to.ptr; p.out_dt = to.dtype;
  p.n_terms = op.sum.n_terms;
  for (int k = 0; k < p.n_terms; ++k) {
    const Tensor& tt = net->tensors[op.sum.term[k]];
    B2R_REQUIRE(tt.ptr, "sum op: unbound term tensor");
    p.term[k] = tt.ptr; p.term_dt[k] = tt.dtype; p.up[k] = op.sum.up[k];
    p.term_C[k] = tt.C; p.term_c_off[k] = op.sum.term_c_off[k];
  }
  p.B = batch; p.H = to.H; p.W = to.W; p.C = to.C; p.relu = op.sum.relu;
  *out = p;
  return B200ROMP_OK;
}

// one op of the plan on `stream`
static int enqueue_op(b200romp_net* net, Op& op, int batch, cudaStream_t stream) {
  ConvParams p;
  if (op.kernel != Kernel::Sum && op.kernel != Kernel::MaxPool) {
    int rc = fill_params(net, op, batch, false, &p);
    if (rc) return rc;
  }
  switch (op.kernel) {
    case Kernel::Sum: {
      SumParams sp;
      int rc = fill_sum_params(net, op, batch, &sp);
      return rc ? rc : launch_fuse_sum(sp, stream);
    }
    case Kernel::MaxPool: {
      const Tensor& ti = net->tensors[op.d.in];
      const Tensor& to = net->tensors[op.d.out];
      B2R_REQUIRE(ti.ptr && to.ptr, "maxpool op: unbound tensor");
      return launch_maxpool3x3s2(ti.ptr, to.ptr, ti.dtype, batch, ti.H, ti.W, ti.C, stream);
    }
    case Kernel::Simt: return launch_conv_simt(p, op.d.ksize, op.d.stride, stream);
    case Kernel::Generic7x7: return launch_conv_generic(p, 7, op.d.stride, stream);
    case Kernel::Deconv4x4: return launch_deconv4x4s2(p, stream);
    case Kernel::Wgmma: return tc_conv_launch(op.tc, p, stream);
    case Kernel::WgmmaStem: return tc_stem_launch(op.tc, p, stream);
    case Kernel::WgmmaConv1d: return tc_conv1d_launch(op.tc, p, stream);
    case Kernel::WgmmaBlock: return tc_block_launch(op.tc, p, stream);
    case Kernel::WgmmaBottleneck: {
      BottleneckMids mids;
      auto mid = [&](int k, int* C) -> __nv_bfloat16* {
        if (!op.parts[k].stored) return nullptr;
        const Tensor& t = net->tensors[op.parts[k].d.out];
        *C = t.C;
        return static_cast<__nv_bfloat16*>(t.ptr);
      };
      mids.t1 = mid(0, &mids.t1_C);
      mids.t2 = mid(1, &mids.t2_C);
      return tc_bottleneck_launch(op.tc, p, mids, stream);
    }
  }
  return B200ROMP_EINVAL;
}

// Pixel-pair folding of a 32->32 3x3 stride-1 conv.  With N = Cout = 32 every MMA still fetches a
// full 128-row A tile from shared memory, so the operand fetch (not the tensor pipe) bounds the layer.  Viewing the NHWC
// tensors as [B, H, W/2, 64] turns the layer into a 64->64 conv whose 3x3 kernel over PAIRS has structured zeros:
// output pair r = pixels (2r, 2r+1) reads pixels 2r-1 .. 2r+2, i.e. pair r-1 (second pixel only), pair r, pair r+1 (first
// pixel only).  W2[dx*32+co][h*32+ci][ky][s+1] = W[co][ci][ky][2s+h-dx+1] when that kx is in 0..2, else 0.  The all-zero
// halves (s=-1,h=0 and s=+1,h=1) are skipped through the plan's kmask: 24 MMAs of N = 64 per 256 pixels instead of 36 of
// N = 32.
static bool fold_eligible(const b200romp_net* net, const Op& op) {
  static const bool off = [] { const char* e = getenv("B200ROMP_TC_NO_FOLD"); return e && e[0] == '1'; }();
  const b200romp_conv_desc& d = op.d;
  const Tensor& ti = net->tensors[d.in];
  const Tensor& to = net->tensors[d.out];
  if (off || d.ksize != 3 || d.stride != 1 || d.upsample != 1 || d.cin != 32 || d.cout != 32) return false;
  if (ti.C != 32 || to.C != 32 || d.in_c_off || d.out_c_off || ti.external || to.external) return false;
  if (ti.dtype != B200ROMP_BF16 || to.dtype != B200ROMP_BF16 || to.nchw || d.pow_channel >= 0 || d.input_norm) return false;
  if (ti.W % 16 != 0 || ti.H % 16 != 0) return false;
  if (d.res >= 0) {
    const Tensor& tr = net->tensors[d.res];
    if (tr.C != 32 || d.res_c_off || d.res_broadcast || tr.dtype != B200ROMP_BF16 || tr.external) return false;
  }
  return true;
}

// in place: [32][32][3][3] weights and [32] bias -> the [64][64][3][3] pair-view weights and [64] bias
static void fold_pixel_pairs(std::vector<float>* w, std::vector<float>* b) {
  std::vector<float> w2((size_t)64 * 64 * 9, 0.f), b2(64);
  for (int dx = 0; dx < 2; ++dx)
    for (int co = 0; co < 32; ++co)
      for (int h = 0; h < 2; ++h)
        for (int ci = 0; ci < 32; ++ci)
          for (int ky = 0; ky < 3; ++ky)
            for (int s = -1; s <= 1; ++s) {
              const int kx = 2 * s + h - dx + 1;
              if (kx < 0 || kx > 2) continue;
              w2[(((size_t)(dx * 32 + co) * 64 + h * 32 + ci) * 3 + ky) * 3 + (s + 1)] = (*w)[(((size_t)co * 32 + ci) * 3 + ky) * 3 + kx];
            }
  for (int i = 0; i < 64; ++i) b2[i] = (*b)[i % 32];
  *w = std::move(w2);
  *b = std::move(b2);
}

// TcConvPlan::kmask of a folded conv
static unsigned fold_kmask() {
  unsigned m = 0;
  for (int t = 0; t < 9; ++t) {
    const int s = t % 3 - 1;
    if (s != -1) m |= 1u << (t * 2 + 0);   // first pixel of the pair is used by s = 0, +1
    if (s != +1) m |= 1u << (t * 2 + 1);   // second pixel by s = -1, 0
  }
  return m;
}

// a bf16 NHWC stride-1 ReLU conv of kernel size `ksize` from cin to cout channels that a fused wgmma kernel may take
static bool is_bf16_relu_conv(const b200romp_net* net, const Op& op, int ksize, int cin, int cout) {
  const b200romp_conv_desc& d = op.d;
  const Tensor& ti = net->tensors[d.in];
  const Tensor& to = net->tensors[d.out];
  return d.ksize == ksize && d.stride == 1 && d.upsample == 1 && d.relu && !d.input_norm && d.pow_channel < 0 &&
         (d.engine == B200ROMP_ENGINE_AUTO || d.engine == B200ROMP_ENGINE_WGMMA) && ti.dtype == B200ROMP_BF16 &&
         to.dtype == B200ROMP_BF16 && !to.nchw && d.cin == cin && d.cout == cout;
}

// how many ops read / write each tensor
static void count_accesses(const b200romp_net* net, std::vector<int>* reads, std::vector<int>* writes) {
  reads->assign(net->tensors.size(), 0);
  writes->assign(net->tensors.size(), 0);
  for (const Op& op : net->ops) {
    ++(*reads)[op.d.in];
    ++(*writes)[op.d.out];
    if (op.kernel == Kernel::Sum)
      for (int k = 0; k < op.sum.n_terms; ++k) ++(*reads)[op.sum.term[k]];
    else if (op.d.res >= 0) ++(*reads)[op.d.res];
  }
}

// `t`, the output of op a and the whole input of op b, can be produced and consumed inside a fused kernel: internal,
// whole-tensor, written by a only and not b's residual.  Ops after b may read it too.
static bool fusable_intermediate(const b200romp_net* net, const Op& a, const Op& b, const std::vector<int>& writes) {
  const int t = a.d.out;
  const Tensor& tt = net->tensors[t];
  return b.d.in == t && b.d.in_c_off == 0 && a.d.out_c_off == 0 && tt.C == a.d.cout && !tt.external && !tt.constant &&
         writes[t] == 1 && b.d.res != t;
}

// A run of consecutive convs that one fused wgmma kernel takes as a single op, the intermediates kept on chip and the input
// read once:
//  - HRNet BasicBlocks relu(conv2(relu(conv1(x))) + x) of 3x3 64->64 convs, or of pixel-pair foldable 32->32 ones, on the
//    block kernel (conv_block_tc.cu);
//  - ResNet Bottlenecks relu(conv3(relu(conv2(relu(conv1(x))))) + x) of 1x1 256->64, 3x3 64->64 and 1x1 64->256 convs (HRNet
//    layer1.1 .. layer1.3) on the Bottleneck kernel (conv_bottleneck_tc.cu).
struct ChainPattern {
  Kernel kernel;
  std::vector<std::array<int, 3>> convs;   // (ksize, cin, cout) of each conv of the chain
  bool fold;                               // the kernel runs on the pixel-pair view: every conv must be fold-eligible
  bool shared_mids;                        // an intermediate may have other readers; the kernel then stores it
  bool (*supported)(const ConvParams& p, bool fold);
};

// Replaces every run of ops that matches `pat` by one op.  Ops i .. i+n-1 fuse when each is a conv as added, of the
// pattern's shape, and all run on one lane; each intermediate is fusable (fusable_intermediate) and, unless the pattern
// shares them, read by nothing else; only the last conv adds a residual, and that is the first conv's input slice; the
// chain's input and output are internal, and the output slice does not overlap the input slice; and the kernel supports the
// fused op.  A caller that binds an intermediate as an external tensor keeps the convs.
static void fuse_chains(b200romp_net* net, const ChainPattern& pat) {
  std::vector<int> reads, writes;
  count_accesses(net, &reads, &writes);
  const size_t n = pat.convs.size();
  std::vector<Op> fused;
  fused.reserve(net->ops.size());
  for (size_t i = 0; i < net->ops.size(); ++i) {
    Op* c = &net->ops[i];
    bool ok = i + n <= net->ops.size();
    for (size_t k = 0; ok && k < n; ++k) {
      const std::array<int, 3>& s = pat.convs[k];
      ok = c[k].kernel == Kernel::Simt && is_bf16_relu_conv(net, c[k], s[0], s[1], s[2]) && c[k].lane == c[0].lane &&
           (!pat.fold || fold_eligible(net, c[k]));
      if (ok && k + 1 < n)
        ok = c[k].d.res < 0 && fusable_intermediate(net, c[k], c[k + 1], writes) && (pat.shared_mids || reads[c[k].d.out] == 1);
    }
    if (ok) {
      const b200romp_conv_desc& first = c[0].d;
      const b200romp_conv_desc& last = c[n - 1].d;
      // in place (output slice over the input slice): the fused kernel stages input halos that neighbouring tiles overwrite
      ok = last.res == first.in && last.res_c_off == first.in_c_off && !last.res_broadcast &&
           !net->tensors[first.in].external && !net->tensors[last.out].external &&
           !(last.out == first.in && slices_overlap(first.in_c_off, first.cin, last.out_c_off, last.cout));
    }
    if (ok) {
      Op f;
      f.kernel = pat.kernel;
      f.d = c[0].d;
      f.d.cout = c[n - 1].d.cout;
      f.d.out = c[n - 1].d.out;
      f.d.out_c_off = c[n - 1].d.out_c_off;
      f.d.res = c[0].d.in;
      f.d.res_c_off = c[n - 1].d.res_c_off;
      f.tc.fold = pat.fold;
      f.lane = c[0].lane;
      ConvParams p;
      fill_params(net, f, 1, true, &p);
      if (pat.supported(p, pat.fold)) {
        for (size_t k = 0; k < n; ++k) {
          f.parts.push_back(std::move(c[k].parts[0]));
          f.parts.back().stored = k + 1 < n && reads[c[k].d.out] > 1;
        }
        fused.push_back(std::move(f));
        i += n - 1;
        continue;
      }
    }
    fused.push_back(std::move(net->ops[i]));
  }
  net->ops = std::move(fused);
}

// Decides op.kernel (and op.tc.fold) of a conv from its descriptor, the requested engine and its tensors' shapes, dtypes and
// flags.  No allocation, no CUDA call: a shape the wgmma engines cannot take runs on the SIMT engine unless the descriptor
// forces B200ROMP_ENGINE_WGMMA.
static int choose_kernel(const b200romp_net* net, int i, Op& op) {
  const b200romp_conv_desc& d = op.d;
  const Tensor& ti = net->tensors[d.in];
  const Tensor& to = net->tensors[d.out];
  if (d.ksize == 7 || d.ksize == 42) {
    op.kernel = d.ksize == 7 ? Kernel::Generic7x7 : Kernel::Deconv4x4;
    return B200ROMP_OK;
  }
  op.kernel = Kernel::Simt;
  const bool forced = d.engine == B200ROMP_ENGINE_WGMMA;
  const bool stem = ti.dtype == B200ROMP_U8 && d.cin == 3 && d.ksize == 3 && d.stride == 2;
  if (!forced && !(d.engine == B200ROMP_ENGINE_TF32 && ti.dtype == B200ROMP_F32) &&
      !(d.engine == B200ROMP_ENGINE_AUTO && (ti.dtype == B200ROMP_BF16 || stem)))
    return B200ROMP_OK;
  ConvParams p;
  fill_params(net, op, net->max_batch, true, &p);
  if (stem) {
    // the stem gathers its u8 input with plain loads (it may be external); its output must be internal
    if (!to.external && d.res < 0 && tc_stem_supported(p, d.ksize, d.stride)) op.kernel = Kernel::WgmmaStem;
  } else if (d.ksize == 13) {
    if (tc_conv1d_supported(p)) op.kernel = Kernel::WgmmaConv1d;   // input tensor map encoded at launch: may be external
  } else if (!ti.external && tc_conv_supported(p, d.ksize, d.stride)) {   // input tensor map encoded at finalize
    op.kernel = Kernel::Wgmma;
    op.tc.fold = fold_eligible(net, op);
  }
  if (forced && op.kernel == Kernel::Simt) {
    set_error("op %d: tensor-core engine forced but shape unsupported", i);
    return B200ROMP_EINVAL;
  }
  return B200ROMP_OK;
}

// Uploads what op's kernel reads and builds its plan.  Every conv gets its bias zero-padded to a multiple of 64 (the wgmma
// epilogues read up to grid_y * NT); only the CUDA-core kernels get the [tap][cin][coutPad] fp32 weights.
static int prepare_op(b200romp_net* net, Op& op) {
  if (op.parts.empty()) return B200ROMP_OK;   // sum, maxpool
  const b200romp_conv_desc& d = op.d;
  // the parts' host weights, freed on return
  std::vector<std::vector<float>> w, b;
  for (Conv& c : op.parts) {
    w.push_back(std::move(c.w));
    b.push_back(std::move(c.b));
    if (op.tc.fold) fold_pixel_pairs(&w.back(), &b.back());
  }
  std::vector<float> bias = b.back();
  op.coutPad = ((int)bias.size() + 63) / 64 * 64;
  bias.resize(op.coutPad, 0.f);
  op.d_bias = static_cast<float*>(upload(bias.data(), bias.size() * sizeof(float), &net->device_allocs));
  if (!op.d_bias) return B200ROMP_ECUDA;
  ConvParams p;
  fill_params(net, op, net->max_batch, true, &p);
  switch (op.kernel) {
    case Kernel::Simt:
    case Kernel::Generic7x7:
    case Kernel::Deconv4x4: {
      const int taps = conv_taps(d.ksize);
      std::vector<float> packed((size_t)taps * d.cin * op.coutPad, 0.f);
      for (int co = 0; co < d.cout; ++co)
        for (int ci = 0; ci < d.cin; ++ci)
          for (int t = 0; t < taps; ++t)   // conv: OIHW; ConvTranspose2d (code 42): PyTorch's [cin][cout][4][4]
            packed[((size_t)t * d.cin + ci) * op.coutPad + co] =
                d.ksize == 42 ? w[0][((size_t)ci * d.cout + co) * taps + t] : w[0][((size_t)co * d.cin + ci) * taps + t];
      op.d_w_simt = static_cast<float*>(upload(packed.data(), packed.size() * sizeof(float), &net->device_allocs));
      return op.d_w_simt ? B200ROMP_OK : B200ROMP_ECUDA;
    }
    case Kernel::Wgmma:
      if (op.tc.fold) op.tc.kmask = fold_kmask();
      return tc_conv_prepare(p, d.ksize, d.stride, w[0].data(), net->sm_count, &op.tc, &net->device_allocs);
    case Kernel::WgmmaStem: return tc_stem_prepare(p, w[0].data(), net->sm_count, &op.tc, &net->device_allocs);
    case Kernel::WgmmaConv1d: return tc_conv1d_prepare(p, w[0].data(), net->sm_count, &op.tc, &net->device_allocs);
    case Kernel::WgmmaBlock:
      return tc_block_prepare(p, w[0].data(), b[0].data(), w[1].data(), net->sm_count, &op.tc, &net->device_allocs);
    case Kernel::WgmmaBottleneck:
      return tc_bottleneck_prepare(p, w[0].data(), b[0].data(), w[1].data(), b[1].data(), w[2].data(), net->sm_count, &op.tc,
                                   &net->device_allocs);
    default: return B200ROMP_OK;
  }
}

int b200romp_net_finalize(b200romp_net* net, int max_batch) {
  B2R_REQUIRE(net && !net->finalized && max_batch > 0, "finalize: bad arguments");
  B2R_CUDA_OK(cudaSetDevice(net->device));
  // before liveness: a fused op's intermediates get no buffer unless other ops read them
  fuse_chains(net, {Kernel::WgmmaBlock, {{3, 64, 64}, {3, 64, 64}}, false, false, tc_block_supported});
  fuse_chains(net, {Kernel::WgmmaBlock, {{3, 32, 32}, {3, 32, 32}}, true, false, tc_block_supported});   // folded to 64
  fuse_chains(net, {Kernel::WgmmaBottleneck, {{1, 256, 64}, {3, 64, 64}, {1, 64, 256}}, false, true,
                    [](const ConvParams& p, bool) { return tc_bottleneck_supported(p); }});
  const int nT = (int)net->tensors.size(), nO = (int)net->ops.size();
  // ---- liveness over the linear op order
  for (int i = 0; i < nO; ++i) {
    const b200romp_conv_desc& d = net->ops[i].d;
    for (int t : op_outputs(net->ops[i])) {
      Tensor& to = net->tensors[t];
      if (to.first_def < 0) to.first_def = i;
      to.last_use = std::max(to.last_use, i);
    }
    net->tensors[d.in].last_use = std::max(net->tensors[d.in].last_use, i);
    if (d.res >= 0) net->tensors[d.res].last_use = std::max(net->tensors[d.res].last_use, i);
    if (net->ops[i].kernel == Kernel::Sum)
      for (int k = 0; k < net->ops[i].sum.n_terms; ++k) {
        Tensor& tt = net->tensors[net->ops[i].sum.term[k]];
        B2R_REQUIRE(tt.external || tt.constant || (tt.first_def >= 0 && tt.first_def < i), "op %d sums tensor %d before it is written", i, net->ops[i].sum.term[k]);
        tt.last_use = std::max(tt.last_use, i);
      }
  }
  for (int i = 0; i < nO; ++i) {
    const b200romp_conv_desc& d = net->ops[i].d;
    const Tensor& ti = net->tensors[d.in];
    B2R_REQUIRE(ti.external || ti.constant || (ti.first_def >= 0 && ti.first_def < i), "op %d reads tensor %d before it is written", i, d.in);
    if (d.res >= 0) {
      const Tensor& tr = net->tensors[d.res];
      B2R_REQUIRE(tr.external || tr.constant || (tr.first_def >= 0 && tr.first_def < i), "op %d adds tensor %d before it is written", i, d.res);
    }
  }
  // ---- buffer planning: exact-size free lists, a buffer is recycled after its tensor's last use
  struct Buf { size_t bytes; size_t offset; };
  std::vector<Buf> bufs;
  std::multimap<size_t, int> free_bufs;
  std::vector<int> tensor_buf(nT, -1);
  std::vector<std::vector<int>> dies_at(nO);
  for (int t = 0; t < nT; ++t) {
    const Tensor& tt = net->tensors[t];
    if (!tt.external && !tt.constant && tt.first_def >= 0) dies_at[tt.last_use].push_back(t);
  }
  size_t total = 0;
  for (int i = 0; i < nO; ++i) {
    for (int t : op_outputs(net->ops[i])) {
      const Tensor& tt = net->tensors[t];
      if (tt.external || tt.constant || tt.first_def != i) continue;
      const size_t bytes = (tt.frame_bytes() * max_batch + 1023) / 1024 * 1024;
      auto it = free_bufs.find(bytes);
      if (it != free_bufs.end()) {
        tensor_buf[t] = it->second;
        free_bufs.erase(it);
      } else {
        bufs.push_back({bytes, total});
        total += bytes;
        tensor_buf[t] = (int)bufs.size() - 1;
      }
    }
    for (int dead : dies_at[i]) free_bufs.insert({bufs[tensor_buf[dead]].bytes, tensor_buf[dead]});
  }
  if (total > 0) {
    B2R_CUDA_OK(cudaMalloc(&net->workspace, total));
    B2R_CUDA_OK(cudaMemset(net->workspace, 0, total));
  }
  net->workspace_bytes = total;
  for (int t = 0; t < nT; ++t)
    if (tensor_buf[t] >= 0) net->tensors[t].ptr = net->workspace + bufs[tensor_buf[t]].offset;
  net->max_batch = max_batch;
  // ---- kernel choice, weight upload, plans
  for (int i = 0; i < nO; ++i) {
    Op& op = net->ops[i];
    int rc = op.kernel == Kernel::Simt ? choose_kernel(net, i, op) : B200ROMP_OK;   // Simt: a conv as added
    if (!rc) rc = prepare_op(net, op);
    if (rc) return rc;
  }
  net->finalized = true;
  return B200ROMP_OK;
}

int b200romp_net_bind(b200romp_net* net, int tensor, void* device_ptr) {
  B2R_REQUIRE(net && tensor >= 0 && tensor < (int)net->tensors.size(), "bind: bad tensor id");
  B2R_REQUIRE(net->tensors[tensor].external, "bind: tensor %d is not external", tensor);
  net->tensors[tensor].ptr = device_ptr;
  return B200ROMP_OK;
}

// Capture-time scheduling: ops are issued in their linear order, each on the stream of its lane.  Cross-lane ordering comes
// from events on the BUFFERS an op touches (workspace buffers are recycled by the liveness planner, so read-after-write,
// write-after-read and write-after-write hazards are all tracked at buffer granularity): the op's lane waits for the last
// writer of everything it reads and for the last writer + all later readers of what it writes.  Inside stream capture the
// events become graph edges.  An op with a cross-lane wait is launched without the programmatic-dependent-launch attribute.
static int enqueue_all_lanes(b200romp_net* net, int batch, cudaStream_t stream) {
  constexpr int L = b200romp_net::kLanes;
  const size_t n = net->ops.size();
  if (net->op_done.size() != n) {
    for (cudaEvent_t e : net->op_done) cudaEventDestroy(e);
    net->op_done.assign(n, nullptr);
    for (auto& e : net->op_done) B2R_CUDA_OK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  }
  if (!net->fork_ev) B2R_CUDA_OK(cudaEventCreateWithFlags(&net->fork_ev, cudaEventDisableTiming));
  for (int l = 1; l < L; ++l)
    if (!net->lane_stream[l]) B2R_CUDA_OK(cudaStreamCreateWithFlags(&net->lane_stream[l], cudaStreamNonBlocking));
  net->lane_stream[0] = stream;
  struct Access { int writer = -1; std::vector<int> readers; };
  std::map<const void*, Access> acc;
  bool lane_used[L] = {true, false, false, false};
  B2R_CUDA_OK(cudaEventRecord(net->fork_ev, stream));
  int rc = B200ROMP_OK;
  for (size_t i = 0; i < n && rc == B200ROMP_OK; ++i) {
    Op& op = net->ops[i];
    const int lane = std::min(std::max(op.lane, 0), L - 1);
    cudaStream_t st = net->lane_stream[lane];
    if (!lane_used[lane]) {
      B2R_CUDA_OK(cudaStreamWaitEvent(st, net->fork_ev, 0));
      lane_used[lane] = true;
    }
    std::vector<const void*> reads, writes;
    for (int t : op_outputs(op)) writes.push_back(net->tensors[t].ptr);
    auto add_read = [&](int t) { if (t >= 0 && !net->tensors[t].constant) reads.push_back(net->tensors[t].ptr); };
    add_read(op.d.in);
    if (op.kernel == Kernel::Sum) for (int k = 0; k < op.sum.n_terms; ++k) add_read(op.sum.term[k]);
    else add_read(op.d.res);
    std::vector<int> deps;
    for (const void* r : reads) { auto it = acc.find(r); if (it != acc.end() && it->second.writer >= 0) deps.push_back(it->second.writer); }
    for (const void* w : writes) { auto it = acc.find(w); if (it != acc.end()) { if (it->second.writer >= 0) deps.push_back(it->second.writer); for (int r : it->second.readers) deps.push_back(r); } }
    std::sort(deps.begin(), deps.end());
    deps.erase(std::unique(deps.begin(), deps.end()), deps.end());
    bool cross = false;
    for (int d : deps) {
      const int dl = std::min(std::max(net->ops[d].lane, 0), L - 1);
      if (dl != lane) { B2R_CUDA_OK(cudaStreamWaitEvent(st, net->op_done[d], 0)); cross = true; }
    }
    g_tc_pdl_override = cross ? 0 : -1;
    rc = enqueue_op(net, op, batch, st);
    g_tc_pdl_override = -1;
    if (rc) break;
    B2R_CUDA_OK(cudaEventRecord(net->op_done[i], st));
    for (const void* r : reads) acc[r].readers.push_back((int)i);
    for (const void* wp : writes) {
      Access& w = acc[wp];
      w.writer = (int)i;
      w.readers.clear();
    }
  }
  // join: the user stream continues after the last op of every lane
  if (rc == B200ROMP_OK) {
    int last[L] = {-1, -1, -1, -1};
    for (size_t i = 0; i < n; ++i) last[std::min(std::max(net->ops[i].lane, 0), L - 1)] = (int)i;
    for (int l = 1; l < L; ++l)
      if (last[l] >= 0) B2R_CUDA_OK(cudaStreamWaitEvent(stream, net->op_done[last[l]], 0));
  }
  return rc;
}

static int enqueue_all(b200romp_net* net, int batch, cudaStream_t stream) {
  for (size_t i = 0; i < net->ops.size(); ++i) {
    int rc = enqueue_op(net, net->ops[i], batch, stream);
    if (rc) return rc;
  }
  return B200ROMP_OK;
}

int b200romp_net_run(b200romp_net* net, int batch, b200romp_stream stream_) {
  B2R_REQUIRE(net && net->finalized, "run: net not finalized");
  B2R_REQUIRE(batch > 0 && batch <= net->max_batch, "run: batch %d outside 1..%d", batch, net->max_batch);
  cudaStream_t stream = (cudaStream_t)stream_;
  B2R_CUDA_OK(cudaSetDevice(net->device));
  if (!net->use_graph || stream == nullptr) return enqueue_all(net, batch, stream);
  b200romp_net::GraphKey key;
  key.batch = batch;
  for (const Tensor& t : net->tensors)
    if (t.external) key.ext.push_back(t.ptr);
  auto it = net->graphs.find(key);
  if (it == net->graphs.end()) {
    cudaGraph_t graph = nullptr;
    cudaError_t e = cudaStreamBeginCapture(stream, cudaStreamCaptureModeThreadLocal);
    if (e != cudaSuccess) {
      cudaGetLastError();
      return enqueue_all(net, batch, stream);   // stream cannot capture (e.g. legacy default stream)
    }
    bool lanes = false;
    if (net->use_lanes)
      for (const Op& op : net->ops) lanes = lanes || op.lane != 0;
    int rc = lanes ? enqueue_all_lanes(net, batch, stream) : enqueue_all(net, batch, stream);
    e = cudaStreamEndCapture(stream, &graph);
    if (rc) {
      if (graph) cudaGraphDestroy(graph);
      return rc;
    }
    B2R_CUDA_OK(e);
    cudaGraphExec_t exec = nullptr;
    B2R_CUDA_OK(cudaGraphInstantiate(&exec, graph, 0));
    cudaGraphDestroy(graph);
    if (net->graphs.size() >= 16) {   // bound the cache: callers normally cycle through a few buffers
      B2R_CUDA_OK(cudaStreamSynchronize(stream));   // an exec may still be running on this stream: never destroy it in flight
      for (auto& kv : net->graphs) cudaGraphExecDestroy(kv.second);
      net->graphs.clear();
    }
    it = net->graphs.insert({key, exec}).first;
  }
  B2R_CUDA_OK(cudaGraphLaunch(it->second, stream));
  return B200ROMP_OK;
}

int b200romp_net_profile(b200romp_net* net, int batch, int iters, float* us_per_op, b200romp_stream stream_) {
  B2R_REQUIRE(net && net->finalized && us_per_op && iters > 0, "profile: bad arguments");
  B2R_REQUIRE(batch > 0 && batch <= net->max_batch, "profile: batch %d outside 1..%d", batch, net->max_batch);
  cudaStream_t stream = (cudaStream_t)stream_;
  B2R_CUDA_OK(cudaSetDevice(net->device));
  const size_t n = net->ops.size();
  std::vector<cudaEvent_t> ev(n + 1);
  for (auto& e : ev) B2R_CUDA_OK(cudaEventCreate(&e));
  std::vector<double> acc(n, 0.0);
  int rc = B200ROMP_OK;
  for (int it = 0; it < iters + 1 && rc == B200ROMP_OK; ++it) {   // pass 0 warms up
    cudaEventRecord(ev[0], stream);
    for (size_t i = 0; i < n && rc == B200ROMP_OK; ++i) {
      rc = enqueue_op(net, net->ops[i], batch, stream);
      cudaEventRecord(ev[i + 1], stream);
    }
    if (rc) break;
    if (cudaStreamSynchronize(stream) != cudaSuccess) { set_error("profile: %s", cudaGetErrorString(cudaGetLastError())); rc = B200ROMP_ECUDA; break; }
    if (it == 0) continue;
    for (size_t i = 0; i < n; ++i) {
      float ms = 0.f;
      cudaEventElapsedTime(&ms, ev[i], ev[i + 1]);
      acc[i] += ms * 1000.0;
    }
  }
  for (auto& e : ev) cudaEventDestroy(e);
  if (rc) return rc;
  for (size_t i = 0; i < n; ++i) us_per_op[i] = (float)(acc[i] / iters);
  return B200ROMP_OK;
}

int b200romp_net_read_tensor(b200romp_net* net, int tensor, int batch, void* dst, b200romp_stream stream) {
  B2R_REQUIRE(net && net->finalized && tensor >= 0 && tensor < (int)net->tensors.size(), "read_tensor: bad arguments");
  const Tensor& t = net->tensors[tensor];
  B2R_REQUIRE(t.ptr != nullptr, "read_tensor: tensor %d has no storage", tensor);
  const size_t bytes = t.frame_bytes() * (t.constant ? 1 : batch);
  B2R_CUDA_OK(cudaMemcpyAsync(dst, t.ptr, bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return B200ROMP_OK;
}

int b200romp_net_describe(b200romp_net* net, char* buf, int len) {
  if (!net || !buf || len <= 0) return B200ROMP_EINVAL;
  std::string s;
  char line[384];
  // the line of one conv; `bracket` describes the kernel that runs it
  auto conv_line = [&](size_t i, const b200romp_conv_desc& d, Kernel kernel, const char* bracket) {
    const Tensor& ti = net->tensors[d.in];
    const Tensor& to = net->tensors[d.out];
    snprintf(line, sizeof(line), "op%03zu %s k%d s%d %4d->%-4d in t%d[%dx%dx%d]+%d out t%d[%dx%dx%d]+%d res t%d up%d relu%d%s\n", i,
             on_wgmma(kernel) ? "wgmma  " : "simt   ", d.ksize, d.stride, d.cin, d.cout, d.in, ti.H, ti.W, ti.C, d.in_c_off, d.out,
             to.H, to.W, to.C, d.out_c_off, d.res, d.upsample, d.relu, bracket);
    s += line;
  };
  for (size_t i = 0; i < net->ops.size(); ++i) {
    const Op& op = net->ops[i];
    const b200romp_conv_desc& d = op.d;
    const Tensor& ti = net->tensors[d.in];
    const Tensor& to = net->tensors[d.out];
    switch (op.kernel) {
      case Kernel::MaxPool:
        snprintf(line, sizeof(line), "op%03zu maxpool 3x3 s2 in t%d[%dx%dx%d] out t%d[%dx%dx%d]\n", i, d.in, ti.H, ti.W, ti.C, d.out, to.H, to.W, to.C);
        s += line;
        break;
      case Kernel::Sum: {
        int n = snprintf(line, sizeof(line), "op%03zu sum     out t%d[%dx%dx%d] = relu%d( t%d", i, op.sum.out, to.H, to.W, to.C, op.sum.relu, op.sum.base);
        for (int k = 0; k < op.sum.n_terms; ++k) n += snprintf(line + n, sizeof(line) - n, " + up%d(t%d)", op.sum.up[k], op.sum.term[k]);
        n += snprintf(line + n, sizeof(line) - n, " )");
        // the kernel follows from the tensors' addresses: named once every tensor of the sum is bound
        bool bound = net->finalized && to.ptr && ti.ptr;
        for (int k = 0; k < op.sum.n_terms; ++k) bound = bound && net->tensors[op.sum.term[k]].ptr;
        SumParams sp;
        if (bound && fill_sum_params(net, op, net->max_batch, &sp) == B200ROMP_OK)
          n += snprintf(line + n, sizeof(line) - n, " [fuse-sum %s]", fuse_sum_kernel_name(sp));
        snprintf(line + n, sizeof(line) - n, "\n");
        s += line;
        break;
      }
      case Kernel::WgmmaBlock: {   // one launch, two convs: a folded block runs both of them on pixel pairs
        const int mid = op.parts[0].d.out;
        const Tensor& tm = net->tensors[mid];
        snprintf(line, sizeof(line),
                 "op%03zu wgmma   block k3 s1 %d->%d->%d in t%d[%dx%dx%d]+%d mid t%d[%dx%dx%d] out t%d[%dx%dx%d]+%d res t%d+%d up1 relu1 "
                 "bias1 bias2 [tc-block grid %d smem %d%s]\n",
                 i, d.cin, d.cin, d.cout, d.in, ti.H, ti.W, ti.C, d.in_c_off, mid, tm.H, tm.W, tm.C, d.out, to.H, to.W, to.C,
                 d.out_c_off, d.res, d.res_c_off, op.tc.grid_x, op.tc.smem_bytes, op.tc.fold ? " conv1 pixel-pairs conv2 pixel-pairs" : "");
        s += line;
        break;
      }
      case Kernel::WgmmaBottleneck:   // one launch, three convs: one line per conv, all with the op's number
        for (size_t k = 0; k < op.parts.size(); ++k) {
          char bracket[96];
          snprintf(bracket, sizeof(bracket), " [tc-bottleneck conv%zu of k1-k3-k1 grid %d smem %d]", k + 1, op.tc.grid_x, op.tc.smem_bytes);
          conv_line(i, op.parts[k].d, op.kernel, bracket);
        }
        break;
      default:
        conv_line(i, d, op.kernel, on_wgmma(op.kernel) ? op.tc.describe().c_str() : "");
    }
  }
  snprintf(line, sizeof(line), "workspace %.1f MiB for max_batch %d\n", net->workspace_bytes / 1048576.0, net->max_batch);
  s += line;
  const int n = (int)std::min<size_t>(s.size(), (size_t)len - 1);
  memcpy(buf, s.data(), n);
  buf[n] = 0;
  return n;
}

int b200romp_net_set_lane(b200romp_net* net, int op, int lane) {
  B2R_REQUIRE(net && !net->finalized && op >= 0 && op < (int)net->ops.size(), "set_lane: bad op id or net already finalized");
  B2R_REQUIRE(lane >= 0 && lane < b200romp_net::kLanes, "set_lane: lane must be 0..%d", b200romp_net::kLanes - 1);
  net->ops[op].lane = lane;
  return B200ROMP_OK;
}

int b200romp_net_num_launches(b200romp_net* net) { return net ? (int)net->ops.size() : 0; }
long long b200romp_net_workspace_bytes(b200romp_net* net) { return net ? (long long)net->workspace_bytes : 0; }

int b200romp_conv2d(const b200romp_conv_desc* d, const float* weight_host, const float* bias_host, const void* in,
                    int in_dtype, int in_H, int in_W, int in_C, void* out, int out_dtype, int out_C, int out_nchw,
                    const void* res, int res_dtype, int batch, b200romp_stream stream) {
  B2R_REQUIRE(d && weight_host && in && out && batch > 0, "conv2d: bad arguments");
  int dev = 0;
  B2R_CUDA_OK(cudaGetDevice(&dev));
  b200romp_net* net = b200romp_net_create(dev);
  if (!net) return B200ROMP_ECUDA;
  int Ho, Wo;
  conv_out_hw(d->ksize, d->stride, in_H, in_W, &Ho, &Wo);   // 13 = Conv1d 1x3, 42 = ConvTranspose2d(4,2,1), 7 = 7x7
  Ho *= d->upsample; Wo *= d->upsample;
  b200romp_conv_desc dd = *d;
  dd.in = b200romp_net_add_tensor(net, in_H, in_W, in_C, in_dtype, 0, 1);
  dd.out = b200romp_net_add_tensor(net, Ho, Wo, out_C, out_dtype, out_nchw, 1);
  dd.res = -1;
  if (res) dd.res = b200romp_net_add_tensor(net, Ho, Wo, out_C, res_dtype, 0, 1);
  int rc = (dd.in < 0 || dd.out < 0) ? B200ROMP_EINVAL : B200ROMP_OK;
  if (!rc) {
    net->tensors[dd.in].ptr = const_cast<void*>(in);
    net->tensors[dd.out].ptr = out;
    if (res) net->tensors[dd.res].ptr = const_cast<void*>(res);
    // stand-alone call: external tensors are allowed on the tensor-core engine because pointers are final
    net->tensors[dd.in].external = net->tensors[dd.out].external = 0;
    if (res) net->tensors[dd.res].external = 0;
    net->tensors[dd.in].constant = true;   // skip "written before read" checks and workspace planning
    net->tensors[dd.out].constant = true;
    if (res) net->tensors[dd.res].constant = true;
    dd.res_c_off = d->out_c_off;
    rc = b200romp_net_add_conv(net, &dd, weight_host, bias_host);
    rc = rc < 0 ? rc : B200ROMP_OK;
  }
  if (!rc) rc = b200romp_net_finalize(net, batch);
  if (!rc) {
    net->use_graph = false;
    rc = b200romp_net_run(net, batch, stream);
  }
  if (!rc) {
    cudaError_t e = cudaStreamSynchronize((cudaStream_t)stream);   // weights are freed below
    if (e != cudaSuccess) {
      set_error("conv2d: %s", cudaGetErrorString(e));
      rc = B200ROMP_ECUDA;
    }
  }
  b200romp_net_destroy(net);
  return rc;
}

}  // extern "C"
