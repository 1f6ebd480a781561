// comm.cu — the two exchange steps of the multi-GPU path inside the C ABI (SURVEY.md §8b/§8e),
// so that a C++ host reaches them without Python:
//   C1  pano_comm_allgather_features  every rank's descriptor sets -> one featureset on every rank
//   C2  pano_comm_allgather_dev       canvas row strips (or any equal-sized device blocks)
// One process (or host thread) per GPU; NCCL over NVLink.  libnccl.so.2 is resolved at run time
// (dlopen), so libpano_b200.so has no link-time dependency on it and single-GPU hosts never load it.
#include "sift.cuh"
#include <dlfcn.h>
#include <nccl.h>      // types and enums only
#include <string.h>
#include <mutex>
#include <vector>

namespace {
struct NcclApi {
  ncclResult_t (*GetUniqueId)(ncclUniqueId*);
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int);
  ncclResult_t (*CommDestroy)(ncclComm_t);
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t);
  ncclResult_t (*GroupStart)();
  ncclResult_t (*GroupEnd)();
  const char* (*GetErrorString)(ncclResult_t);
  bool ok = false;
};
NcclApi g_nccl;
std::mutex g_nccl_mu;

bool load_nccl(std::string* why) {
  std::lock_guard<std::mutex> lock(g_nccl_mu);
  if (g_nccl.ok) return true;
  void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  if (!h) { *why = dlerror(); return false; }
#define NCCL_SYM(field, name) do { *(void**)&g_nccl.field = dlsym(h, name); if (!g_nccl.field) { *why = "missing symbol " name; return false; } } while (0)
  NCCL_SYM(GetUniqueId, "ncclGetUniqueId"); NCCL_SYM(CommInitRank, "ncclCommInitRank"); NCCL_SYM(CommDestroy, "ncclCommDestroy");
  NCCL_SYM(AllGather, "ncclAllGather"); NCCL_SYM(GroupStart, "ncclGroupStart"); NCCL_SYM(GroupEnd, "ncclGroupEnd");
  NCCL_SYM(GetErrorString, "ncclGetErrorString");
#undef NCCL_SYM
  g_nccl.ok = true;
  return true;
}
}  // namespace

struct pano_comm {
  pano_ctx* ctx = nullptr;
  ncclComm_t comm = nullptr;
  int world = 1, rank = 0;
  bool owned = false;
};

#define PANO_NCCL(c, call)                                                                              \
  do {                                                                                                  \
    ncclResult_t _r = (call);                                                                           \
    if (_r != ncclSuccess) return ctx_fail((c)->ctx, PANO_ERR_CUDA, "NCCL error %s at %s", g_nccl.GetErrorString(_r), #call); \
  } while (0)

int featureset_build_dev(pano_ctx* ctx, int n_images, const int* n_kp, const float* const* d_desc,
                         const double* const* d_coor, pano_featureset** out);   // engine.cu

extern "C" {

int pano_comm_unique_id(unsigned char id[128]) {
  std::string why;
  if (!id) return PANO_ERR_INVALID;
  if (!load_nccl(&why)) return ctx_fail(nullptr, PANO_ERR_NO_DEVICE, "libnccl.so.2 not available: %s", why.c_str());
  static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
  ncclUniqueId u;
  if (g_nccl.GetUniqueId(&u) != ncclSuccess) return ctx_fail(nullptr, PANO_ERR_CUDA, "ncclGetUniqueId failed");
  memcpy(id, &u, 128);
  return PANO_OK;
}

int pano_comm_create(pano_ctx* ctx, int world, int rank, const unsigned char id[128], pano_comm** out) {
  ctx_enter(ctx);
  if (!ctx || !out || !id || world < 1 || rank < 0 || rank >= world) return PANO_ERR_INVALID;
  *out = nullptr;
  std::string why;
  if (!load_nccl(&why)) return ctx_fail(ctx, PANO_ERR_NO_DEVICE, "libnccl.so.2 not available: %s", why.c_str());
  pano_comm* c = new pano_comm;
  c->ctx = ctx; c->world = world; c->rank = rank; c->owned = true;
  ncclUniqueId u;
  memcpy(&u, id, 128);
  ncclResult_t r = g_nccl.CommInitRank(&c->comm, world, u, rank);
  if (r != ncclSuccess) { int rc = ctx_fail(ctx, PANO_ERR_CUDA, "ncclCommInitRank: %s", g_nccl.GetErrorString(r)); delete c; return rc; }
  *out = c;
  return PANO_OK;
}

int pano_comm_adopt(pano_ctx* ctx, void* nccl_comm, int world, int rank, pano_comm** out) {
  ctx_enter(ctx);
  if (!ctx || !out || !nccl_comm || world < 1 || rank < 0 || rank >= world) return PANO_ERR_INVALID;
  std::string why;
  if (!load_nccl(&why)) return ctx_fail(ctx, PANO_ERR_NO_DEVICE, "libnccl.so.2 not available: %s", why.c_str());
  pano_comm* c = new pano_comm;
  c->ctx = ctx; c->comm = (ncclComm_t)nccl_comm; c->world = world; c->rank = rank; c->owned = false;
  *out = c;
  return PANO_OK;
}

void pano_comm_destroy(pano_comm* c) {
  if (!c) return;
  ctx_enter(c->ctx);
  if (c->owned && c->comm) { cudaStreamSynchronize(c->ctx->stream); g_nccl.CommDestroy(c->comm); }
  delete c;
}

int pano_comm_world(const pano_comm* c) { return c ? c->world : PANO_ERR_INVALID; }
int pano_comm_rank(const pano_comm* c) { return c ? c->rank : PANO_ERR_INVALID; }

int pano_comm_allgather_dev(pano_comm* c, const void* d_send, void* d_recv, size_t bytes_per_rank) {
  if (!c || !d_send || !d_recv) return PANO_ERR_INVALID;
  ctx_enter(c->ctx);
  PANO_NCCL(c, g_nccl.AllGather(d_send, d_recv, bytes_per_rank, ncclUint8, c->comm, c->ctx->stream));
  return PANO_OK;
}

// C1.  Image k of the n_images_total images is owned by rank k mod world (the image loop of
// calc_feature dealt round-robin, stitcherbase.cc:14); `local` holds this rank's images in
// ascending k.  Counts first (one small all-gather + host read), then one padded all-gather each
// of the descriptor rows and the coordinates, then an import on the device: no host staging.
int pano_comm_allgather_features(pano_comm* c, pano_featureset* local, int n_images_total, pano_featureset** all) {
  if (!c || !all || n_images_total <= 0) return PANO_ERR_INVALID;
  pano_ctx* ctx = c->ctx;
  ctx_enter(ctx);
  *all = nullptr;
  const int W = c->world, R = c->rank;
  const int per_rank = (n_images_total + W - 1) / W;
  const int mine = (n_images_total - R + W - 1) / W;                 // images k = R, R+W, ...
  if ((mine > 0 && !local) || (local && local->n_images != mine))
    return ctx_fail(ctx, PANO_ERR_INVALID, "allgather_features: rank %d owns %d of %d images, featureset has %d", R, mine,
                    n_images_total, local ? local->n_images : 0);
  int rc = 0;
  if (local && (rc = featureset_sync_counts(local))) return rc;
  // ---- counts
  DevBuf<int> d_cnt_send, d_cnt_all;
  if ((rc = d_cnt_send.alloc(ctx, per_rank)) || (rc = d_cnt_all.alloc(ctx, (size_t)per_rank * W))) return rc;
  std::vector<int> cnt_mine(per_rank, 0);
  for (int q = 0; q < mine; ++q) cnt_mine[q] = local->h_count[q];
  if ((rc = ctx_put(ctx, d_cnt_send, cnt_mine.data(), per_rank * sizeof(int)))) return rc;
  PANO_NCCL(c, g_nccl.AllGather(d_cnt_send, d_cnt_all, per_rank, ncclInt32, c->comm, ctx->stream));
  std::vector<int> cnt_all((size_t)per_rank * W);
  PANO_CUDA(ctx, cudaMemcpyAsync(cnt_all.data(), d_cnt_all, cnt_all.size() * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  PANO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  d_cnt_send.reset(); d_cnt_all.reset();   // before the payload buffers, which may take their blocks
  std::vector<int> counts(n_images_total);
  size_t pad = 1;
  for (int r = 0; r < W; ++r) {
    size_t rows = 0;
    for (int q = 0; r + q * W < n_images_total; ++q) { counts[r + q * W] = cnt_all[(size_t)r * per_rank + q]; rows += cnt_all[(size_t)r * per_rank + q]; }
    pad = std::max(pad, rows);
  }
  // ---- payload
  DevBuf<float> d_send, d_all;
  DevBuf<double> c_send, c_all;
  if ((rc = d_send.alloc(ctx, pad * 128)) || (rc = d_all.alloc(ctx, pad * W * 128)) || (rc = c_send.alloc(ctx, pad * 2)) ||
      (rc = c_all.alloc(ctx, pad * W * 2)))
    return rc;
  {
    // this rank's rows into the send buffers: one launch for all images
    std::vector<void*> dsts; std::vector<const void*> srcs; std::vector<size_t> sizes;
    size_t off = 0;
    for (int q = 0; q < mine; ++q) {
      const size_t nq = (size_t)local->h_count[q];
      if (nq) {
        dsts.push_back(d_send + off * 128); srcs.push_back(local->d_desc + local->base[q] * 128); sizes.push_back(nq * 128 * sizeof(float));
        if (local->d_coor) { dsts.push_back(c_send + off * 2); srcs.push_back(local->d_coor + local->base[q] * 2); sizes.push_back(nq * 2 * sizeof(double)); }
      }
      off += nq;
    }
    if ((rc = ctx_copy_blocks(ctx, (int)dsts.size(), dsts.data(), srcs.data(), sizes.data()))) return rc;
  }
  {
    ncclResult_t r1 = g_nccl.GroupStart();
    ncclResult_t r2 = g_nccl.AllGather(d_send, d_all, pad * 128, ncclFloat32, c->comm, ctx->stream);
    ncclResult_t r3 = g_nccl.AllGather(c_send, c_all, pad * 2, ncclFloat64, c->comm, ctx->stream);
    ncclResult_t r4 = g_nccl.GroupEnd();
    if (r1 != ncclSuccess || r2 != ncclSuccess || r3 != ncclSuccess || r4 != ncclSuccess)
      return ctx_fail(ctx, PANO_ERR_CUDA, "NCCL all-gather of the descriptor sets failed");
  }
  {
    std::vector<const float*> pd(n_images_total);
    std::vector<const double*> pc(n_images_total);
    for (int r = 0; r < W; ++r) {
      size_t off = 0;
      for (int k = r; k < n_images_total; k += W) {
        pd[k] = d_all + ((size_t)r * pad + off) * 128;
        pc[k] = c_all + ((size_t)r * pad + off) * 2;
        off += counts[k];
      }
    }
    return featureset_build_dev(ctx, n_images_total, counts.data(), pd.data(), pc.data(), all);   // the buffers go after the import
  }
}

}  // extern "C"
