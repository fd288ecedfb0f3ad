// Multi-GPU form of the path behind the C ABI (SURVEY 8b / 8e): ONE process drives every visible GPU.
//
// The reference has no distributed layer; pairs are independent, so the batch is split contiguously over the
// devices (equal counts), every device runs K0..K2 on its share from its own stream, and ONE ncclAllGather of
// the compact result segments (include/b200align.h: b2a_batch_compact_*) reassembles the per-pair results on
// every device; device 0's copy is decoded into the caller's host arrays (b2a_gathered_fetch).  The segment size
// is agreed on the host (one process: a max over the per-device sizes, no collective).
//
// NCCL is bound at run time (dlopen of libnccl.so.2: ncclCommInitAll, ncclAllGather, group calls), so the library
// still loads on a machine without NCCL; if it cannot be found the segments are gathered onto device 0 with
// peer-to-peer copies over NVLink instead (same bytes, same decode) and b2a_multi_exchange_kind() says so.
#include <cuda_runtime.h>
#include <dlfcn.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

#include "../../include/b200align.h"

namespace {

typedef void* nccl_comm_t;
typedef int (*fn_comm_init_all)(nccl_comm_t*, int, const int*);
typedef int (*fn_comm_destroy)(nccl_comm_t);
typedef int (*fn_all_gather)(const void*, void*, size_t, int, nccl_comm_t, cudaStream_t);
typedef int (*fn_group)(void);
typedef const char* (*fn_err_string)(int);
constexpr int kNcclUint8 = 1;  // ncclDataType_t: ncclInt8 0, ncclUint8 1 (nccl.h)

}  // namespace

struct b2a_multi {
  std::vector<int> devs;
  std::vector<b2a_engine*> eng;
  std::vector<cudaStream_t> streams;
  std::vector<void*> seg_local, seg_all;
  uint64_t seg_cap = 0;
  void* nccl = nullptr;
  fn_comm_init_all comm_init_all = nullptr;
  fn_comm_destroy comm_destroy = nullptr;
  fn_all_gather all_gather = nullptr;
  fn_group group_start = nullptr, group_end = nullptr;
  fn_err_string err_string = nullptr;
  std::vector<nccl_comm_t> comms;
  bool use_nccl = false;
  std::string err;
  int fail(int code, const std::string& what) {
    err = what;
    return code;
  }
};

extern "C" {

const char* b2a_multi_last_error(const b2a_multi* m) { return m ? m->err.c_str() : "null multi-engine"; }

const char* b2a_multi_exchange_kind(const b2a_multi* m) {
  if (!m) return "none";
  if (m->devs.size() < 2) return "single device: no exchange";
  return m->use_nccl ? "ncclAllGather (libnccl.so.2, ncclCommInitAll)" : "cudaMemcpyPeerAsync onto device 0 (libnccl.so.2 not found)";
}

int32_t b2a_multi_destroy(b2a_multi* m) {
  if (!m) return B2A_OK;
  for (size_t d = 0; d < m->devs.size(); ++d) {
    cudaSetDevice(m->devs[d]);
    if (d < m->streams.size() && m->streams[d]) cudaStreamSynchronize(m->streams[d]);
    if (d < m->comms.size() && m->comms[d] && m->comm_destroy) m->comm_destroy(m->comms[d]);
    if (d < m->eng.size() && m->eng[d]) b2a_engine_destroy(m->eng[d]);
    if (d < m->seg_local.size() && m->seg_local[d]) cudaFree(m->seg_local[d]);
    if (d < m->seg_all.size() && m->seg_all[d]) cudaFree(m->seg_all[d]);
    if (d < m->streams.size() && m->streams[d]) cudaStreamDestroy(m->streams[d]);
  }
  if (m->nccl) dlclose(m->nccl);
  delete m;
  return B2A_OK;
}

int32_t b2a_multi_create(b2a_multi** out, const int32_t* device_ids, int32_t n_devices) {
  if (!out) return B2A_E_INVALID;
  *out = nullptr;
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0) return B2A_E_NO_DEVICE;
  if (n_devices <= 0) n_devices = count;  // all visible devices
  if (n_devices > count) return B2A_E_NO_DEVICE;
  b2a_multi* m = new b2a_multi();
  for (int d = 0; d < n_devices; ++d) m->devs.push_back(device_ids ? device_ids[d] : d);
  const size_t nd = m->devs.size();
  m->eng.assign(nd, nullptr);
  m->streams.assign(nd, nullptr);
  m->seg_local.assign(nd, nullptr);
  m->seg_all.assign(nd, nullptr);
  for (size_t d = 0; d < nd; ++d) {
    const int rc = b2a_engine_create(&m->eng[d], m->devs[d]);
    if (rc) {
      b2a_multi_destroy(m);
      return rc;
    }
    cudaSetDevice(m->devs[d]);
    if (cudaStreamCreateWithFlags(&m->streams[d], cudaStreamNonBlocking) != cudaSuccess) {
      b2a_multi_destroy(m);
      return B2A_E_CUDA;
    }
    b2a_engine_set_stream(m->eng[d], m->streams[d]);
    b2a_engine_set_pipeline(m->eng[d], 0);  // shards are staged whole; the devices themselves run side by side
  }
  if (nd > 1) {
    const char* names[] = {getenv("B2A_NCCL_PATH"), "libnccl.so.2", "libnccl.so"};
    for (const char* nm : names) {
      if (!nm || !*nm) continue;
      m->nccl = dlopen(nm, RTLD_NOW | RTLD_LOCAL);
      if (m->nccl) break;
    }
    if (m->nccl) {
      m->comm_init_all = (fn_comm_init_all)dlsym(m->nccl, "ncclCommInitAll");
      m->comm_destroy = (fn_comm_destroy)dlsym(m->nccl, "ncclCommDestroy");
      m->all_gather = (fn_all_gather)dlsym(m->nccl, "ncclAllGather");
      m->group_start = (fn_group)dlsym(m->nccl, "ncclGroupStart");
      m->group_end = (fn_group)dlsym(m->nccl, "ncclGroupEnd");
      m->err_string = (fn_err_string)dlsym(m->nccl, "ncclGetErrorString");
      if (m->comm_init_all && m->comm_destroy && m->all_gather && m->group_start && m->group_end) {
        m->comms.assign(nd, nullptr);
        const int rc = m->comm_init_all(m->comms.data(), (int)nd, m->devs.data());
        if (rc == 0) {
          m->use_nccl = true;
        } else {
          m->comms.clear();
        }
      }
    }
    if (!m->use_nccl) {  // peer-copy gather: device 0 must be able to read its peers
      cudaSetDevice(m->devs[0]);
      for (size_t d = 1; d < nd; ++d) {
        int can = 0;
        cudaDeviceCanAccessPeer(&can, m->devs[0], m->devs[d]);
        if (can) cudaDeviceEnablePeerAccess(m->devs[d], 0);  // (cudaMemcpyPeerAsync works without it, through the host)
      }
      cudaGetLastError();
    }
  }
  *out = m;
  return B2A_OK;
}

int32_t b2a_multi_device_count(const b2a_multi* m) { return m ? (int32_t)m->devs.size() : 0; }

int32_t b2a_multi_align_batch(b2a_multi* m, int32_t mode, const b2a_scoring* scoring, const b2a_pairs* pairs,
                              b2a_results* results, b2a_stats* stats) {
  if (!m || !scoring || !pairs || !results) return B2A_E_INVALID;
  const size_t nd = m->devs.size();
  const uint64_t n = pairs->n_pairs;
  if (nd == 1 || n < nd) {
    cudaSetDevice(m->devs[0]);
    const int rc = b2a_align_batch(m->eng[0], mode, scoring, pairs, results, stats);
    if (rc) m->err = b2a_last_error(m->eng[0]);
    return rc;
  }
  // contiguous split with equal counts (SURVEY 8e)
  const uint64_t per = (n + nd - 1) / nd;
  std::vector<uint64_t> lo(nd), hi(nd), seg_bytes(nd, 0);
  std::vector<int> rcs(nd, B2A_OK);
  std::vector<b2a_stats> dstats(nd);
  std::vector<std::vector<uint64_t>> xoff(nd), yoff(nd);
  for (size_t d = 0; d < nd; ++d) {
    lo[d] = std::min<uint64_t>(n, d * per);
    hi[d] = std::min<uint64_t>(n, lo[d] + per);
  }
  // every device: stage (H2D of its shard) + run + the size of its result segment, side by side
  {
    std::vector<std::thread> pool;
    for (size_t d = 0; d < nd; ++d) {
      pool.emplace_back([&, d]() {
        cudaSetDevice(m->devs[d]);
        const uint64_t nc = hi[d] - lo[d];
        uint64_t bmin = ~0ull, bmax = 0;
        for (uint64_t p = lo[d]; p < hi[d]; ++p) {
          const uint64_t bb = pairs->blob_bytes, xo = pairs->x_off[p], yo = pairs->y_off[p];
          if (xo > bb || pairs->x_len[p] > bb - xo || yo > bb || pairs->y_len[p] > bb - yo) {
            rcs[d] = B2A_E_INVALID;
            return;
          }
          bmin = std::min(bmin, std::min(xo, yo));
          bmax = std::max(bmax, std::max(xo + pairs->x_len[p], yo + pairs->y_len[p]));
        }
        if (bmin > bmax) bmin = bmax = 0;
        xoff[d].resize(nc);
        yoff[d].resize(nc);
        for (uint64_t i = 0; i < nc; ++i) {
          xoff[d][i] = pairs->x_off[lo[d] + i] - bmin;
          yoff[d][i] = pairs->y_off[lo[d] + i] - bmin;
        }
        b2a_pairs sub{pairs->seq_blob + bmin, xoff[d].data(), pairs->x_len + lo[d], yoff[d].data(), pairs->y_len + lo[d],
                      bmax - bmin, nc};
        int rc = b2a_batch_stage(m->eng[d], mode, scoring, &sub);
        if (rc == B2A_OK) rc = b2a_batch_run(m->eng[d]);
        if (rc == B2A_OK) rc = b2a_batch_fetch(m->eng[d], nullptr, &dstats[d]);  // waits; reports a failing pair
        if (rc == B2A_OK) rc = b2a_batch_compact_bytes(m->eng[d], &seg_bytes[d]);
        rcs[d] = rc;
      });
    }
    for (auto& t : pool) t.join();
  }
  for (size_t d = 0; d < nd; ++d)
    if (rcs[d]) return m->fail(rcs[d], rcs[d] == B2A_E_INVALID && !*b2a_last_error(m->eng[d])
                                          ? std::string("sequence offset/length outside seq_blob")
                                          : std::string("device ") + std::to_string(m->devs[d]) + ": " + b2a_last_error(m->eng[d]));
  uint64_t seg = 0;
  for (uint64_t v : seg_bytes) seg = std::max(seg, v);
  seg = (seg + 255) & ~255ull;
  if (seg > m->seg_cap) {
    for (size_t d = 0; d < nd; ++d) {
      cudaSetDevice(m->devs[d]);
      if (m->seg_local[d]) cudaFree(m->seg_local[d]);
      if (m->seg_all[d]) cudaFree(m->seg_all[d]);
      m->seg_local[d] = m->seg_all[d] = nullptr;
      const bool need_all = m->use_nccl || d == 0;
      if (cudaMalloc(&m->seg_local[d], seg + seg / 8) != cudaSuccess ||
          (need_all && cudaMalloc(&m->seg_all[d], (seg + seg / 8) * nd) != cudaSuccess)) {
        m->seg_cap = 0;
        return m->fail(B2A_E_CUDA, "cudaMalloc of the result segments failed");
      }
    }
    m->seg_cap = seg + seg / 8;
    seg = m->seg_cap & ~255ull;
  } else {
    seg = m->seg_cap & ~255ull;
  }
  for (size_t d = 0; d < nd; ++d) {
    cudaSetDevice(m->devs[d]);
    const int rc = b2a_batch_compact_into(m->eng[d], m->seg_local[d], seg);
    if (rc) return m->fail(rc, b2a_last_error(m->eng[d]));
  }
  if (m->use_nccl) {  // the one collective of the path
    int rc = m->group_start();
    for (size_t d = 0; d < nd && rc == 0; ++d) {
      cudaSetDevice(m->devs[d]);
      rc = m->all_gather(m->seg_local[d], m->seg_all[d], (size_t)seg, kNcclUint8, m->comms[d], m->streams[d]);
    }
    const int rc2 = m->group_end();
    if (rc || rc2)
      return m->fail(B2A_E_CUDA, std::string("ncclAllGather failed: ") + (m->err_string ? m->err_string(rc ? rc : rc2) : "?"));
  } else {
    for (size_t d = 0; d < nd; ++d) {  // device d's segment -> its slot in device 0's gather buffer
      cudaSetDevice(m->devs[d]);
      cudaStreamSynchronize(m->streams[d]);
    }
    cudaSetDevice(m->devs[0]);
    for (size_t d = 0; d < nd; ++d) {
      const cudaError_t ce = cudaMemcpyPeerAsync(reinterpret_cast<uint8_t*>(m->seg_all[0]) + d * seg, m->devs[0],
                                                 m->seg_local[d], m->devs[d], seg, m->streams[0]);
      if (ce != cudaSuccess) return m->fail(B2A_E_CUDA, std::string("cudaMemcpyPeerAsync: ") + cudaGetErrorString(ce));
    }
  }
  cudaSetDevice(m->devs[0]);
  uint64_t got = 0, d2h = 0;
  int rc = b2a_gathered_fetch(m->eng[0], m->seg_all[0], seg, (uint32_t)nd, results, &got, &d2h);
  if (rc) return m->fail(rc, b2a_last_error(m->eng[0]));
  if (got != n) return m->fail(B2A_E_STATE, "gathered segments do not hold the whole batch");
  for (size_t d = 1; d < nd; ++d) {  // the other devices' gathers finish before their buffers are reused
    cudaSetDevice(m->devs[d]);
    cudaStreamSynchronize(m->streams[d]);
  }
  if (stats) {
    std::memset(stats, 0, sizeof(*stats));
    for (size_t d = 0; d < nd; ++d) {
      stats->cells += dstats[d].cells;
      stats->h2d_bytes += dstats[d].h2d_bytes;
      stats->traceback_bytes += dstats[d].traceback_bytes;
      stats->pack_ms = std::max(stats->pack_ms, dstats[d].pack_ms);
      stats->fill_ms = std::max(stats->fill_ms, dstats[d].fill_ms);
      stats->walk_ms = std::max(stats->walk_ms, dstats[d].walk_ms);
      stats->kernel_launches += dstats[d].kernel_launches;
      stats->waves = std::max(stats->waves, dstats[d].waves);
    }
    stats->d2h_bytes = d2h;
    stats->fill_lanes_per_pair = dstats[0].fill_lanes_per_pair;
    stats->fill_rows_per_lane = dstats[0].fill_rows_per_lane;
  }
  return B2A_OK;
}

}  // extern "C"
