// Descriptor-network executor.  The host (dcr_b200/nets.py) describes a network once as a list of ops over
// numbered activation tensors and uploaded parameters -- mirroring the nn.Module structure of the reference models
// (torchvision ResNet-50 trunk of SSCD, dino_vits.VisionTransformer, metrics/inception.InceptionV3) -- and then
// calls dcr_net_forward(images_u8, n) per batch; everything between the uint8 image batch and the fp32 descriptor
// rows runs here as hand-written kernels on one stream.  Replaces `model(samples)` in
// utils_ret.py:751 / embedding_search/utils.py:101 / metrics/fid.py:126.
#include <cuda_bf16.h>

#include <cstring>
#include <memory>
#include <vector>

#include "dcr_internal.cuh"
#include "host_util.cuh"
#include "image_in.cuh"

namespace dcr {

struct NetTensor {
  long long rows_per_image;
  int C;
  __nv_bfloat16* ptr;
  long long plane_stride;   // elements
  bool owned = true;        // false: a reshaped view of another tensor's buffer (net_alias_tensor)
  int alias_of = -1;        // the tensor whose buffer a view shares
};

// Uploaded weights and per-channel tables: read-only after upload, shared by a network and its forks.
struct ParamStore {
  std::vector<void*> ptrs;
  ~ParamStore() {
    for (void* p : ptrs) cudaFree(p);
  }
};

struct NetOp {
  int kind;
  int i[24];
  float f[12];
};

struct Net {
  int max_batch = 0;
  int planes = 1;
  int terms = 1;
  int exact = 0;   // convolutions / linear layers accumulate in float64 (needs planes == 3)
  int out_dim = 0;
  float* out_f32 = nullptr;   // [max_batch, out_dim]
  std::vector<NetTensor> tensors;
  std::shared_ptr<ParamStore> store = std::make_shared<ParamStore>();
  std::vector<NetOp> ops;
  size_t bytes_allocated = 0;
};

namespace {
const int kTermA[6] = {0, 0, 1, 1, 0, 2};
const int kTermW[6] = {0, 1, 0, 1, 2, 0};

// The input prefix of IM2COL_U8, STEM_S2D and STEM_ROWS: ints [out_t, IH, IW, crop_y, crop_x, H, W], floats [mean[3],
// std[3], post_scale, post_shift]; the resizing form adds RH, RW at ints [rs, rs + 1] and rscale at floats [8] (unset
// arguments are zero: no resizing).
int input_source(const NetOp& op, int rs, const uint8_t* images, const float* images_f32, ImageSource* s) {
  const int* a = op.i;
  const bool f32 = images_f32 != nullptr;
  s->img = images;
  s->img_f32 = images_f32;
  // fp32 input: the tensor is the transformed crop itself ([B,3,H,W]: no crop offset)
  s->IH = f32 ? a[5] : a[1];
  s->IW = f32 ? a[6] : a[2];
  s->crop_y = f32 ? 0 : a[3];
  s->crop_x = f32 ? 0 : a[4];
  s->H = a[5];
  s->W = a[6];
  s->rscale = op.f[8];
  s->RH = s->rscale == 0.f ? s->H : a[rs];
  s->RW = s->rscale == 0.f ? s->W : a[rs + 1];
  for (int c = 0; c < 3; ++c) {
    s->mean[c] = op.f[c];
    s->std[c] = op.f[3 + c];
  }
  s->post_scale = op.f[6];
  s->post_shift = op.f[7];
  DCR_REQUIRE(s->crop_y >= 0 && s->crop_x >= 0 && s->crop_y + s->H <= s->IH && s->crop_x + s->W <= s->IW,
              "net_forward: %d x %d crop at (%d, %d) outside the %d x %d image", s->H, s->W, s->crop_y, s->crop_x, s->IH, s->IW);
  return 0;
}
}

int net_create(int max_batch, int planes, Net** out) {
  DCR_REQUIRE(max_batch >= 1 && max_batch <= 65536, "net_create: bad max_batch %d", max_batch);
  DCR_REQUIRE(planes >= 1 && planes <= 3, "net_create: planes must be 1..3");
  if (!device_info()) return -2;
  Net* n = new Net();
  n->max_batch = max_batch;
  n->planes = planes;
  n->terms = planes == 1 ? 1 : (planes == 2 ? 3 : 6);
  *out = n;
  return 0;
}

int net_set_exact(Net* n, int on) {
  DCR_REQUIRE(n != nullptr, "net_set_exact: null handle");
  DCR_REQUIRE(!on || n->planes == 3, "net_set_exact: exact arithmetic needs the 3-plane (fp32) tensor format");
  n->exact = on ? 1 : 0;
  return 0;
}

void net_destroy(Net* n) {
  if (!n) return;
  for (auto& t : n->tensors)
    if (t.owned) cudaFree(t.ptr);
  if (n->out_f32) cudaFree(n->out_f32);
  delete n;
}

// A second executor for the same network: own activation buffers and output rows, the SAME uploaded parameters.
// Two forward passes (two batches, two streams) can then be in flight at once -- the persistent kernels of one fill the
// SMs the other leaves idle at its wave tails (tools/dual_stream.py: +15 % images/s at batch 256).
int net_fork(const Net* src, Net** out) {
  DCR_REQUIRE(src != nullptr && out != nullptr, "net_fork: null argument");
  Net* n = new Net();
  n->max_batch = src->max_batch;
  n->planes = src->planes;
  n->terms = src->terms;
  n->exact = src->exact;
  n->store = src->store;
  n->ops = src->ops;
  for (const NetTensor& s : src->tensors) {
    NetTensor t = s;
    if (s.alias_of >= 0) {
      t.ptr = n->tensors[s.alias_of].ptr;
    } else {
      const size_t bytes = static_cast<size_t>(t.plane_stride) * n->planes * 2 + 1024;
      void* p = nullptr;
      cudaError_t e = cudaMalloc(&p, bytes);
      if (e == cudaSuccess) e = cudaMemset(p, 0, bytes);
      if (e != cudaSuccess) {
        if (p) cudaFree(p);
        net_destroy(n);
        return set_error(-2, "net_fork: %s", cudaGetErrorString(e));
      }
      t.ptr = static_cast<__nv_bfloat16*>(p);
      n->bytes_allocated += bytes;
    }
    n->tensors.push_back(t);
  }
  if (src->out_dim > 0) {
    if (int rc = net_set_output(n, src->out_dim)) {
      net_destroy(n);
      return rc;
    }
  }
  *out = n;
  return 0;
}

int net_add_tensor(Net* n, long long rows_per_image, int C) {
  DCR_REQUIRE(n && rows_per_image >= 1 && C >= 8 && C % 8 == 0, "net_add_tensor: bad shape (%lld, %d)", rows_per_image, C);
  NetTensor t;
  t.rows_per_image = rows_per_image;
  t.C = C;
  t.plane_stride = static_cast<long long>(n->max_batch) * rows_per_image * C;
  const size_t bytes = static_cast<size_t>(t.plane_stride) * n->planes * 2 + 1024;   // slack: TMA boxes may read past
  void* p = nullptr;
  DCR_CUDA_CHECK(cudaMalloc(&p, bytes));
  DCR_CUDA_CHECK(cudaMemset(p, 0, bytes));
  t.ptr = static_cast<__nv_bfloat16*>(p);
  n->bytes_allocated += bytes;
  n->tensors.push_back(t);
  return static_cast<int>(n->tensors.size()) - 1;
}

// A second shape for an existing activation buffer: same elements per image, other (rows, channels) factorisation
// (flatten of the NHWC feature map in front of a Linear layer: VGG-16's classifier in metrics/ipr.py:139-141).
int net_alias_tensor(Net* n, int src, long long rows_per_image, int C) {
  DCR_REQUIRE(n && src >= 0 && src < static_cast<int>(n->tensors.size()), "net_alias_tensor: bad source tensor");
  const NetTensor& s = n->tensors[src];
  DCR_REQUIRE(rows_per_image >= 1 && C >= 8 && C % 8 == 0 && rows_per_image * C == s.rows_per_image * s.C,
              "net_alias_tensor: (%lld, %d) does not hold the %lld elements per image of the source", rows_per_image, C,
              s.rows_per_image * s.C);
  NetTensor t = s;
  t.rows_per_image = rows_per_image;
  t.C = C;
  t.owned = false;
  t.alias_of = s.alias_of >= 0 ? s.alias_of : src;
  n->tensors.push_back(t);
  return static_cast<int>(n->tensors.size()) - 1;
}

int net_tensor(const Net* n, int t, void** ptr, long long* plane_stride) {
  DCR_REQUIRE(n && t >= 0 && t < static_cast<int>(n->tensors.size()), "net_tensor: bad tensor id %d", t);
  *ptr = n->tensors[t].ptr;
  *plane_stride = n->tensors[t].plane_stride;
  return 0;
}

int net_add_param(Net* n, const void* host, size_t bytes) {
  DCR_REQUIRE(n && host && bytes > 0, "net_add_param: bad arguments");
  void* p = nullptr;
  DCR_CUDA_CHECK(cudaMalloc(&p, bytes + 256));
  DCR_CUDA_CHECK(cudaMemcpy(p, host, bytes, cudaMemcpyHostToDevice));
  n->bytes_allocated += bytes;
  n->store->ptrs.push_back(p);
  return static_cast<int>(n->store->ptrs.size()) - 1;
}

int net_set_output(Net* n, int dim) {
  DCR_REQUIRE(n && dim >= 4 && dim % 4 == 0, "net_set_output: dim %d must be a positive multiple of 4", dim);
  if (n->out_f32) cudaFree(n->out_f32);
  n->out_dim = dim;
  DCR_CUDA_CHECK(cudaMalloc(reinterpret_cast<void**>(&n->out_f32), static_cast<size_t>(n->max_batch) * dim * 4 + 256));
  return 0;
}

int net_add_op(Net* n, int kind, const int* iargs, int ni, const float* fargs, int nf) {
  DCR_REQUIRE(n && kind >= 0 && kind < NET_OP_COUNT, "net_add_op: unknown op kind %d", kind);
  DCR_REQUIRE(ni >= 0 && ni <= 24 && nf >= 0 && nf <= 12, "net_add_op: too many arguments");
  NetOp op;
  memset(&op, 0, sizeof(op));
  op.kind = kind;
  for (int j = 0; j < ni; ++j) op.i[j] = iargs[j];
  for (int j = 0; j < nf; ++j) op.f[j] = fargs[j];
  auto tensor_ok = [&](int id, bool optional) { return (optional && id < 0) || (id >= 0 && id < (int)n->tensors.size()); };
  auto param_ok = [&](int id, bool optional) { return (optional && id < 0) || (id >= 0 && id < (int)n->store->ptrs.size()); };
  switch (kind) {
    case NET_OP_IM2COL_U8:
      DCR_REQUIRE(((ni == 12 && nf == 8) || (ni == 14 && nf == 9)) && tensor_ok(op.i[0], false), "im2col_u8 op: bad args");
      break;
    case NET_OP_STEM_S2D:
      DCR_REQUIRE(((ni == 7 && nf == 8) || (ni == 9 && nf == 9)) && tensor_ok(op.i[0], false), "stem_s2d op: bad args");
      break;
    case NET_OP_CONV:
      DCR_REQUIRE((ni == 18 || ni == 20) && tensor_ok(op.i[0], false) && tensor_ok(op.i[1], true) && param_ok(op.i[5], false) &&
                      param_ok(op.i[12], true) && param_ok(op.i[13], true) && tensor_ok(op.i[14], true),
                  "conv op: bad args");
      break;
    case NET_OP_MAXPOOL:
    case NET_OP_AVGPOOL: DCR_REQUIRE(ni == 9 && tensor_ok(op.i[0], false) && tensor_ok(op.i[1], false), "pool op: bad args"); break;
    case NET_OP_GEM: DCR_REQUIRE(ni == 5 && nf == 2 && tensor_ok(op.i[0], false) && tensor_ok(op.i[1], true), "gem op: bad args"); break;
    case NET_OP_GAP: DCR_REQUIRE(ni == 5 && tensor_ok(op.i[0], false) && tensor_ok(op.i[1], true), "gap op: bad args"); break;
    case NET_OP_LAYERNORM:
      DCR_REQUIRE(ni == 8 && nf == 1 && tensor_ok(op.i[0], false) && tensor_ok(op.i[1], true) && param_ok(op.i[4], false) &&
                      param_ok(op.i[5], false),
                  "layernorm op: bad args");
      break;
    case NET_OP_VIT_TOKENS:
      DCR_REQUIRE(ni == 6 && tensor_ok(op.i[0], false) && tensor_ok(op.i[1], false) && param_ok(op.i[4], false) &&
                      param_ok(op.i[5], false),
                  "vit_tokens op: bad args");
      break;
    case NET_OP_ATTENTION:
      DCR_REQUIRE((ni == 5 || ni == 6) && nf == 1 && tensor_ok(op.i[0], false) && tensor_ok(op.i[1], false), "attention op: bad args");
      break;
    case NET_OP_EMBED:
      DCR_REQUIRE(ni == 6 && tensor_ok(op.i[0], false) && param_ok(op.i[3], false) && param_ok(op.i[4], false), "embed op: bad args");
      break;
    case NET_OP_L2NORM_OUT: DCR_REQUIRE(nf == 1, "l2norm op: bad args"); break;
    case NET_OP_STEM_ROWS:
      DCR_REQUIRE(((ni == 7 && nf == 8) || (ni == 9 && nf == 9)) && tensor_ok(op.i[0], false) && n->planes == 1, "stem_rows op: bad args");
      break;
    case NET_OP_STEM_CONV:
      DCR_REQUIRE((ni == 7 || ni == 8) && tensor_ok(op.i[0], false) && tensor_ok(op.i[1], false) && param_ok(op.i[4], false) &&
                      param_ok(op.i[5], true) && param_ok(op.i[6], true) && n->planes == 1,
                  "stem_conv op: bad args");
      break;
    default: break;
  }
  n->ops.push_back(op);
  return static_cast<int>(n->ops.size()) - 1;
}

int net_forward(Net* n, const uint8_t* images, int B, float* out, cudaStream_t stream, const float* images_f32) {
  DCR_REQUIRE(n && (images || images_f32) && out, "net_forward: null argument");
  const bool f32 = images_f32 != nullptr;
  DCR_REQUIRE(B >= 0 && B <= n->max_batch, "net_forward: batch %d exceeds max_batch %d", B, n->max_batch);
  DCR_REQUIRE(n->out_f32 && n->out_dim > 0, "net_forward: output not configured");
  if (B == 0) return 0;
  const int P = n->planes;
  auto conv_desc = [&](const NetOp& cop) {
    const int* a = cop.i;
    const NetTensor& in = n->tensors[a[0]];
    ConvGemmDesc d;
    d.in = in.ptr;
    d.in_plane_stride = in.plane_stride;
    d.B = B; d.H = a[2]; d.W = a[3]; d.C = a[4]; d.ld_in = in.C;
    d.weight = static_cast<const __nv_bfloat16*>(n->store->ptrs[a[5]]);
    d.N = a[6]; d.kh = a[7]; d.kw = a[8]; d.stride = a[9]; d.pad_h = a[10]; d.pad_w = a[11];
    if (a[18] > 0) {   // overlapping-window view: a[18] = elements per stored pixel, a[19] = stored pixels per row
      d.in_stride_w = a[18];
      d.in_stride_h = static_cast<long long>(a[18]) * a[19];
      d.in_stride_n = in.rows_per_image * in.C;
    }
    const int cpad = (d.C + 63) / 64 * 64;
    d.w_plane_stride = static_cast<long long>(d.N) * d.kh * d.kw * cpad;
    d.n_terms = n->terms;
    for (int t = 0; t < n->terms; ++t) { d.term_a[t] = kTermA[t]; d.term_w[t] = kTermW[t]; }
    d.scale = a[12] >= 0 ? static_cast<const float*>(n->store->ptrs[a[12]]) : nullptr;
    d.bias = a[13] >= 0 ? static_cast<const float*>(n->store->ptrs[a[13]]) : nullptr;
    if (a[14] >= 0) {
      const NetTensor& r = n->tensors[a[14]];
      d.res = r.ptr; d.ld_res = r.C; d.res_planes = P; d.res_plane_stride = r.plane_stride;
    }
    d.act = a[15];
    d.exact = n->exact;
    if (a[1] >= 0) {
      NetTensor& o = n->tensors[a[1]];
      d.out = o.ptr; d.ld_out = o.C; d.out_col_off = a[16]; d.out_planes = P; d.out_plane_stride = o.plane_stride;
    }
    // fp32 output rows are the op's own N wide: [B, N] for a head on pooled features, [B * T, N] = [B, T * N] for a
    // per-token projection (CLIP text tower)
    if (a[17]) { d.out_f32 = n->out_f32; d.ld_out_f32 = d.N; }
    return d;
  };
  for (size_t oi = 0; oi < n->ops.size(); ++oi) {
    const NetOp& op = n->ops[oi];
    const int* a = op.i;
    int rc = 0;
    switch (op.kind) {
      case NET_OP_IM2COL_U8: {
        NetTensor& t = n->tensors[a[0]];
        ImageSource src;
        rc = input_source(op, 12, images, images_f32, &src);
        if (rc == 0) rc = im2col_u8(src, B, a[7], a[8], a[9], a[10], a[11], t.ptr, t.plane_stride, P, stream);
        break;
      }
      case NET_OP_STEM_S2D: {
        NetTensor& t = n->tensors[a[0]];
        ImageSource src;
        rc = input_source(op, 7, images, images_f32, &src);
        if (rc == 0) rc = stem_s2d_u8(src, B, t.ptr, t.plane_stride, P, stream);
        break;
      }
      case NET_OP_STEM_ROWS: {
        ImageSource src;
        rc = input_source(op, 7, images, images_f32, &src);
        if (rc == 0) rc = stem_rows(src, B, n->tensors[a[0]].ptr, stream);
        break;
      }
      case NET_OP_STEM_CONV: {
        const NetTensor& in = n->tensors[a[0]];
        NetTensor& o = n->tensors[a[1]];
        const long long out_rows = a[7] ? static_cast<long long>((a[2] - 1) / 2 + 1) * ((a[3] - 1) / 2 + 1) : static_cast<long long>(a[2]) * a[3];
        DCR_REQUIRE(in.rows_per_image == 2 * stem_fused_plane_units(a[2], a[3]) && in.C == 8 && o.C == 64 && o.rows_per_image == out_rows,
                    "stem_conv op: tensor shapes do not match the %d x %d output", a[2], a[3]);
        rc = stem_conv(in.ptr, B, a[2], a[3], static_cast<const __nv_bfloat16*>(n->store->ptrs[a[4]]),
                       a[5] >= 0 ? static_cast<const float*>(n->store->ptrs[a[5]]) : nullptr,
                       a[6] >= 0 ? static_cast<const float*>(n->store->ptrs[a[6]]) : nullptr, o.ptr, stream, a[7]);
        break;
      }
      case NET_OP_CONV: {
        ConvGemmDesc d = conv_desc(op);
        // peephole: conv3 (1x1 expand + residual + ReLU) directly followed by the next block's conv1 (1x1 reduce + ReLU)
        // on its output -> one fused kernel that never re-reads the expanded activation (bottleneck_fuse.cu)
        if (oi + 1 < n->ops.size() && n->ops[oi + 1].kind == NET_OP_CONV) {
          const ConvGemmDesc d2 = conv_desc(n->ops[oi + 1]);
          const DeviceInfo* di = device_info();
          if (di && expand_reduce_eligible(d, d2, di->max_smem_optin)) {
            rc = expand_reduce(d, d2, stream);
            ++oi;   // the second convolution is done
            break;
          }
        }
        {
          const DeviceInfo* di = device_info();
          if (di && expand_only_eligible(d, di->max_smem_optin)) {
            rc = expand_only(d, stream);
            break;
          }
        }
        rc = conv_gemm(d, stream);
        break;
      }
      case NET_OP_MAXPOOL:
      case NET_OP_AVGPOOL: {
        const NetTensor& in = n->tensors[a[0]];
        NetTensor& o = n->tensors[a[1]];
        rc = pool2d(op.kind == NET_OP_MAXPOOL, in.ptr, in.plane_stride, o.ptr, o.plane_stride, P, B, a[2], a[3], a[4],
                    a[5], a[6], a[7], o.C, a[8], stream);
        break;
      }
      case NET_OP_GEM:
      case NET_OP_GAP: {
        const NetTensor& in = n->tensors[a[0]];
        __nv_bfloat16* op_out = a[1] >= 0 ? n->tensors[a[1]].ptr : nullptr;
        const long long ops = a[1] >= 0 ? n->tensors[a[1]].plane_stride : 0;
        rc = reduce_hw(op.kind == NET_OP_GEM, in.ptr, in.plane_stride, P, B, a[2], a[3], op.f[0], op.f[1], op_out, ops,
                       a[4] ? n->out_f32 : nullptr, stream);
        break;
      }
      case NET_OP_LAYERNORM: {
        const NetTensor& in = n->tensors[a[0]];
        __nv_bfloat16* op_out = a[1] >= 0 ? n->tensors[a[1]].ptr : nullptr;
        const long long ops = a[1] >= 0 ? n->tensors[a[1]].plane_stride : 0;
        rc = layernorm(in.ptr, in.plane_stride, P, B * a[2], a[3], static_cast<long long>(a[6]) * a[3],
                       static_cast<const float*>(n->store->ptrs[a[4]]), static_cast<const float*>(n->store->ptrs[a[5]]), op.f[0],
                       op_out, ops, a[7] ? n->out_f32 : nullptr, stream);
        break;
      }
      case NET_OP_VIT_TOKENS: {
        const NetTensor& in = n->tensors[a[0]];
        NetTensor& o = n->tensors[a[1]];
        rc = vit_tokens(in.ptr, in.plane_stride, static_cast<const float*>(n->store->ptrs[a[4]]),
                        static_cast<const float*>(n->store->ptrs[a[5]]), o.ptr, o.plane_stride, P, B, a[2], a[3], stream);
        break;
      }
      case NET_OP_ATTENTION: {
        const NetTensor& in = n->tensors[a[0]];
        NetTensor& o = n->tensors[a[1]];
        rc = attention(in.ptr, in.plane_stride, o.ptr, o.plane_stride, P, B, a[2], a[3], a[4], op.f[0], stream, a[5]);
        break;
      }
      case NET_OP_EMBED: {   // the network input is int32 token ids [B, T] (passed through the `images` pointer)
        NetTensor& o = n->tensors[a[0]];
        DCR_REQUIRE(images != nullptr && !f32, "net_forward: this network takes int32 token ids");
        rc = embed_tokens(reinterpret_cast<const int*>(images), B, a[1], a[2], static_cast<const float*>(n->store->ptrs[a[3]]), a[5],
                          static_cast<const float*>(n->store->ptrs[a[4]]), o.ptr, o.plane_stride, P, stream);
        break;
      }
      case NET_OP_L2NORM_OUT: rc = l2_normalize(n->out_f32, B, n->out_dim, op.f[0], stream); break;
      default: rc = set_error(-1, "net_forward: unknown op kind %d", op.kind);
    }
    if (rc != 0) return rc;
  }
  DCR_CUDA_CHECK(cudaMemcpyAsync(out, n->out_f32, static_cast<size_t>(B) * n->out_dim * 4, cudaMemcpyDeviceToDevice, stream));
  return 0;
}

}  // namespace dcr
