// Multi-GPU form of the path behind the C ABI (SURVEY 8b / 8e): ONE process drives every visible GPU.
//
// The reference has no distributed layer; pairs are independent, so the batch is split contiguously over the
// devices (equal counts), every device runs its share from its own stream, and ONE ncclAllGather of the compact
// result segments (include/b200align.h: b2a_batch_compact_*) reassembles the per-pair results on every device;
// device 0's copy is decoded into the caller's host arrays (b2a_gathered_fetch).  The segment size is agreed on
// the host (one process: a max over the per-device sizes, no collective).  One driver (run_split) does the split,
// the per-device threads, the exchange and the decode for every aligner; only the job a device runs on its share
// differs: K0..K2 (Aligner), K4 + K3 (banded::Aligner), or a score-only call whose outputs go straight to the
// caller's host arrays (no ops, so nothing to exchange).
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
#include <functional>
#include <set>
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
  bool repeated = false;  // a device is listed more than once: one engine per entry, peer copies onto entry 0
  // the engines holding the last call's Myers hit list (b2a_multi_myers_batch with a listing; empty after any other
  // call): entry d's pairs [lo, hi) of the caller's list and its hit count, in pair order
  struct HeldHits {
    size_t d;
    uint64_t lo, hi, hits;
  };
  std::vector<HeldHits> myers_held;
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
  if (m->repeated) return "cudaMemcpyPeerAsync onto entry 0 (a device is listed more than once: no NCCL communicator)";
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
  if (!device_ids && n_devices > count) return B2A_E_NO_DEVICE;
  for (int d = 0; device_ids && d < n_devices; ++d)  // a list may repeat a device, but each must exist
    if (device_ids[d] < 0 || device_ids[d] >= count) return B2A_E_NO_DEVICE;
  b2a_multi* m = new b2a_multi();
  for (int d = 0; d < n_devices; ++d) m->devs.push_back(device_ids ? device_ids[d] : d);
  const size_t nd = m->devs.size();
  // ncclCommInitAll takes each device once; a list that repeats one runs every entry on its own engine and stream
  m->repeated = std::set<int>(m->devs.begin(), m->devs.end()).size() != nd;
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
  if (nd > 1 && !m->repeated) {
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
  }
  if (nd > 1 && !m->use_nccl) {  // peer-copy gather: device 0 must be able to read its peers
    cudaSetDevice(m->devs[0]);
    for (size_t d = 1; d < nd; ++d) {
      if (m->devs[d] == m->devs[0]) continue;
      int can = 0;
      cudaDeviceCanAccessPeer(&can, m->devs[0], m->devs[d]);
      if (can) cudaDeviceEnablePeerAccess(m->devs[d], 0);  // (cudaMemcpyPeerAsync works without it, through the host)
    }
    cudaGetLastError();
  }
  *out = m;
  return B2A_OK;
}

int32_t b2a_multi_device_count(const b2a_multi* m) { return m ? (int32_t)m->devs.size() : 0; }

}  // extern "C"

namespace {

// One device's share of a batch: pairs [lo, hi) of the caller's list, over the part of the blob they use.
struct Share {
  uint64_t lo = 0, hi = 0;
  std::vector<uint64_t> xoff, yoff;
  b2a_pairs pairs{};
};

// What an engine runs on the whole batch (fewer pairs than devices) or on one share; a share job leaves a full
// result on its engine when the driver exchanges (b2a_batch_compact_*), else it has written the caller's arrays.
typedef std::function<int32_t(b2a_engine*)> WholeJob;
typedef std::function<int32_t(b2a_engine*, const Share&, b2a_stats*)> ShareJob;

// the per-pair status array of a share: a b2a_results holding only status + lo (NULL without a status array, so a
// failing pair still fails the call as on one engine)
b2a_results status_slice(const b2a_results* r, uint64_t lo) {
  b2a_results s{};
  if (r && r->status) s.status = r->status + lo;
  return s;
}

// Cells, bytes and launches add up over the devices; kernel times and waves are the slowest device's; the shape
// fields are device 0's.
void merge_stats(const std::vector<b2a_stats>& ds, uint64_t exchange_d2h, b2a_stats* out) {
  std::memset(out, 0, sizeof(*out));
  for (const b2a_stats& s : ds) {
    out->cells += s.cells;
    out->h2d_bytes += s.h2d_bytes;
    out->d2h_bytes += s.d2h_bytes;
    out->traceback_bytes += s.traceback_bytes;
    out->pack_ms = std::max(out->pack_ms, s.pack_ms);
    out->fill_ms = std::max(out->fill_ms, s.fill_ms);
    out->walk_ms = std::max(out->walk_ms, s.walk_ms);
    out->band_ms = std::max(out->band_ms, s.band_ms);
    out->kernel_launches += s.kernel_launches;
    out->waves = std::max(out->waves, s.waves);
  }
  out->d2h_bytes += exchange_d2h;
  out->fill_lanes_per_pair = ds[0].fill_lanes_per_pair;
  out->fill_rows_per_lane = ds[0].fill_rows_per_lane;
}

// The one multi-GPU driver.  A batch of fewer pairs than devices runs `whole` on device 0.  Otherwise the pair list
// is split contiguously into equal counts and every device runs `job` on its share from its own thread; with
// `exchange` each device's result is compacted into a segment, the segments are all-gathered (or peer-copied onto
// entry 0) and device 0's copy is decoded into `results`.  Per-pair statuses travel outside the segments: each job
// fetched its own slice of results->status.
int32_t run_split(b2a_multi* m, const b2a_pairs* pairs, b2a_results* results, b2a_stats* stats, bool exchange,
                  const WholeJob& whole, const ShareJob& job) {
  const size_t nd = m->devs.size();
  const uint64_t n = pairs->n_pairs;
  m->myers_held.clear();
  if (nd == 1 || n < nd) {
    cudaSetDevice(m->devs[0]);
    const int rc = whole(m->eng[0]);
    if (rc) m->err = b2a_last_error(m->eng[0]);
    return rc;
  }
  // contiguous split with equal counts (SURVEY 8e)
  const uint64_t per = (n + nd - 1) / nd;
  std::vector<Share> sh(nd);
  std::vector<uint64_t> seg_bytes(nd, 0);
  std::vector<int> rcs(nd, B2A_OK);
  std::vector<char> bad_range(nd, 0);
  std::vector<b2a_stats> dstats(nd);
  for (size_t d = 0; d < nd; ++d) {
    sh[d].lo = std::min<uint64_t>(n, d * per);
    sh[d].hi = std::min<uint64_t>(n, sh[d].lo + per);
  }
  // every device: its share (H2D, kernels, fetch) and the size of its result segment, side by side
  {
    std::vector<std::thread> pool;
    for (size_t d = 0; d < nd; ++d) {
      pool.emplace_back([&, d]() {
        cudaSetDevice(m->devs[d]);
        Share& s = sh[d];
        const uint64_t nc = s.hi - s.lo;
        uint64_t bmin = ~0ull, bmax = 0;
        for (uint64_t p = s.lo; p < s.hi; ++p) {
          const uint64_t bb = pairs->blob_bytes, xo = pairs->x_off[p], yo = pairs->y_off[p];
          if (xo > bb || pairs->x_len[p] > bb - xo || yo > bb || pairs->y_len[p] > bb - yo) {
            bad_range[d] = 1;
            rcs[d] = B2A_E_INVALID;
            return;
          }
          bmin = std::min(bmin, std::min(xo, yo));
          bmax = std::max(bmax, std::max(xo + pairs->x_len[p], yo + pairs->y_len[p]));
        }
        if (bmin > bmax) bmin = bmax = 0;
        s.xoff.resize(nc);
        s.yoff.resize(nc);
        for (uint64_t i = 0; i < nc; ++i) {
          s.xoff[i] = pairs->x_off[s.lo + i] - bmin;
          s.yoff[i] = pairs->y_off[s.lo + i] - bmin;
        }
        s.pairs = b2a_pairs{pairs->seq_blob + bmin, s.xoff.data(), pairs->x_len + s.lo, s.yoff.data(),
                            pairs->y_len + s.lo, bmax - bmin, nc};
        int rc = job(m->eng[d], s, &dstats[d]);
        if (rc == B2A_OK && exchange) rc = b2a_batch_compact_bytes(m->eng[d], &seg_bytes[d]);
        rcs[d] = rc;
      });
    }
    for (auto& t : pool) t.join();
  }
  for (size_t d = 0; d < nd; ++d)
    if (rcs[d]) return m->fail(rcs[d], bad_range[d] ? std::string("sequence offset/length outside seq_blob")
                                                    : std::string("device ") + std::to_string(m->devs[d]) + ": " +
                                                          b2a_last_error(m->eng[d]));
  if (!exchange) {  // the jobs wrote the caller's host arrays themselves
    if (stats) merge_stats(dstats, 0, stats);
    return B2A_OK;
  }
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
  b2a_results body = *results;
  body.status = nullptr;  // the jobs fetched the statuses; the segments carry none
  int rc = b2a_gathered_fetch(m->eng[0], m->seg_all[0], seg, (uint32_t)nd, &body, &got, &d2h);
  if (rc) return m->fail(rc, b2a_last_error(m->eng[0]));
  if (got != n) return m->fail(B2A_E_STATE, "gathered segments do not hold the whole batch");
  for (size_t d = 1; d < nd; ++d) {  // the other devices' gathers finish before their buffers are reused
    cudaSetDevice(m->devs[d]);
    cudaStreamSynchronize(m->streams[d]);
  }
  if (stats) merge_stats(dstats, d2h, stats);
  return B2A_OK;
}

// A hint list is outside input: the rules of the single engine's check, and match_off / path_off ascending over
// the whole batch, hold before anything is sliced (a share's pointers are built from these offsets).
int32_t check_hints(b2a_multi* m, const b2a_pairs* pairs, const b2a_band_hints* h) {
  const uint64_t n = pairs->n_pairs;
  if (!h->match_off || (!h->match_xy && n && h->match_off[n]))
    return m->fail(B2A_E_INVALID, "banded hints: match_off / match_xy missing");
  if (h->path_off && (h->allowed_mismatches >= 0 || h->use_lcskpp_union))
    return m->fail(B2A_E_INVALID, "banded hints: a match path excludes allowed_mismatches / use_lcskpp_union");
  if (h->path_off && !h->path_idx && n && h->path_off[n]) return m->fail(B2A_E_INVALID, "banded hints: path_idx missing");
  for (uint64_t p = 0; p < n; ++p) {
    if (h->match_off[p + 1] < h->match_off[p]) return m->fail(B2A_E_INVALID, "banded hints: match_off not ascending");
    if (h->path_off && h->path_off[p + 1] < h->path_off[p])
      return m->fail(B2A_E_INVALID, "banded hints: path_off not ascending");
  }
  return B2A_OK;
}

// the hints of pairs [lo, hi): offsets rebased to the share's first pair (path indices are per pair: unchanged)
struct HintShare {
  std::vector<uint64_t> moff, poff;
  b2a_band_hints h{};
  HintShare(const b2a_band_hints* src, uint64_t lo, uint64_t hi) {
    h = *src;
    moff.resize(hi - lo + 1);
    for (uint64_t p = lo; p <= hi; ++p) moff[p - lo] = src->match_off[p] - src->match_off[lo];
    h.match_off = moff.data();
    h.match_xy = src->match_xy ? src->match_xy + 2 * src->match_off[lo] : nullptr;
    if (src->path_off) {
      poff.resize(hi - lo + 1);
      for (uint64_t p = lo; p <= hi; ++p) poff[p - lo] = src->path_off[p] - src->path_off[lo];
      h.path_off = poff.data();
      h.path_idx = src->path_idx ? src->path_idx + src->path_off[lo] : nullptr;
    }
  }
};

// score-only outputs: score, xend, yend and status, each at the share's offset; the rest must be NULL
bool score_only_outputs_ok(b2a_multi* m, const b2a_results* r) {
  if (r && (r->xstart || r->ystart || r->ops || r->ops_off || r->clip_len)) {
    m->fail(B2A_E_INVALID, "a score-only batch has only score, xend, yend and status: xstart, ystart, ops, ops_off and "
                           "clip_len must be NULL");
    return false;
  }
  return true;
}

b2a_results score_slice(const b2a_results* r, uint64_t lo) {
  b2a_results s{};
  s.score = r->score ? r->score + lo : nullptr;
  s.xend = r->xend ? r->xend + lo : nullptr;
  s.yend = r->yend ? r->yend + lo : nullptr;
  s.status = r->status ? r->status + lo : nullptr;
  return s;
}

}  // namespace

extern "C" {

int32_t b2a_multi_align_batch(b2a_multi* m, int32_t mode, const b2a_scoring* scoring, const b2a_pairs* pairs,
                              b2a_results* results, b2a_stats* stats) {
  if (!m || !scoring || !pairs || !results) return B2A_E_INVALID;
  return run_split(
      m, pairs, results, stats, true,
      [&](b2a_engine* e) { return b2a_align_batch(e, mode, scoring, pairs, results, stats); },
      [&](b2a_engine* e, const Share& s, b2a_stats* st) {
        b2a_results r = status_slice(results, s.lo);
        int rc = b2a_batch_stage(e, mode, scoring, &s.pairs);
        if (rc == B2A_OK) rc = b2a_batch_run(e);
        if (rc == B2A_OK) rc = b2a_batch_fetch(e, r.status ? &r : nullptr, st);  // waits; reports a failing pair
        return rc;
      });
}

int32_t b2a_multi_align_batch_banded(b2a_multi* m, int32_t mode, const b2a_scoring* scoring, uint32_t k, uint32_t w,
                                     const b2a_pairs* pairs, const b2a_band_hints* hints, b2a_results* results,
                                     b2a_stats* stats) {
  if (!m || !scoring || !pairs || !results) return B2A_E_INVALID;
  if (hints) {
    const int rc = check_hints(m, pairs, hints);
    if (rc) return rc;
  }
  return run_split(
      m, pairs, results, stats, true,
      [&](b2a_engine* e) {
        return hints ? b2a_align_batch_banded_hinted(e, mode, scoring, k, w, pairs, hints, results, stats)
                     : b2a_align_batch_banded(e, mode, scoring, k, w, pairs, results, stats);
      },
      [&](b2a_engine* e, const Share& s, b2a_stats* st) {  // the result stays on the engine for the compaction
        b2a_results r = status_slice(results, s.lo);
        b2a_results* rp = r.status ? &r : nullptr;
        if (!hints) return b2a_align_batch_banded(e, mode, scoring, k, w, &s.pairs, rp, st);
        const HintShare hs(hints, s.lo, s.hi);
        return b2a_align_batch_banded_hinted(e, mode, scoring, k, w, &s.pairs, &hs.h, rp, st);
      });
}

int32_t b2a_multi_align_batch_scores(b2a_multi* m, int32_t mode, const b2a_scoring* scoring, const b2a_pairs* pairs,
                                     b2a_results* results, b2a_stats* stats) {
  if (!m || !scoring || !pairs) return B2A_E_INVALID;
  if (!score_only_outputs_ok(m, results)) return B2A_E_INVALID;
  return run_split(
      m, pairs, results, stats, false,
      [&](b2a_engine* e) { return b2a_align_batch_scores(e, mode, scoring, pairs, results, stats); },
      [&](b2a_engine* e, const Share& s, b2a_stats* st) {
        b2a_results r = results ? score_slice(results, s.lo) : b2a_results{};
        return b2a_align_batch_scores(e, mode, scoring, &s.pairs, results ? &r : nullptr, st);
      });
}

int32_t b2a_multi_align_batch_banded_scores(b2a_multi* m, int32_t mode, const b2a_scoring* scoring, uint32_t k,
                                            uint32_t w, const b2a_pairs* pairs, const b2a_band_hints* hints,
                                            b2a_results* results, b2a_stats* stats) {
  if (!m || !scoring || !pairs) return B2A_E_INVALID;
  if (!score_only_outputs_ok(m, results)) return B2A_E_INVALID;
  if (hints) {
    const int rc = check_hints(m, pairs, hints);
    if (rc) return rc;
  }
  return run_split(
      m, pairs, results, stats, false,
      [&](b2a_engine* e) { return b2a_align_batch_banded_scores(e, mode, scoring, k, w, pairs, hints, results, stats); },
      [&](b2a_engine* e, const Share& s, b2a_stats* st) {
        b2a_results r = results ? score_slice(results, s.lo) : b2a_results{};
        if (!hints) return b2a_align_batch_banded_scores(e, mode, scoring, k, w, &s.pairs, nullptr, results ? &r : nullptr, st);
        const HintShare hs(hints, s.lo, s.hi);
        return b2a_align_batch_banded_scores(e, mode, scoring, k, w, &s.pairs, &hs.h, results ? &r : nullptr, st);
      });
}

int32_t b2a_multi_levenshtein_batch(b2a_multi* m, uint32_t k, const b2a_pairs* pairs, uint32_t* distance,
                                    b2a_stats* stats) {
  if (!m || !pairs || (!distance && pairs->n_pairs)) return B2A_E_INVALID;
  return run_split(
      m, pairs, nullptr, stats, false, [&](b2a_engine* e) { return b2a_levenshtein_batch(e, k, pairs, distance, stats); },
      [&](b2a_engine* e, const Share& s, b2a_stats* st) {
        return b2a_levenshtein_batch(e, k, &s.pairs, distance + s.lo, st);
      });
}

int32_t b2a_multi_hamming_batch(b2a_multi* m, const b2a_pairs* pairs, uint32_t* distance, uint32_t* status,
                                b2a_stats* stats) {
  if (!m || !pairs || (!distance && pairs->n_pairs)) return B2A_E_INVALID;
  if (!status && m->devs.size() > 1) {
    // a pair of unequal lengths fails the call; a share would name it by its index in the share, so the whole batch
    // is checked here first (offsets, then lengths, in the single engine's order) and the caller's index reported
    for (uint64_t p = 0; p < pairs->n_pairs; ++p) {
      const uint64_t bb = pairs->blob_bytes, xo = pairs->x_off[p], yo = pairs->y_off[p];
      if (xo > bb || pairs->x_len[p] > bb - xo || yo > bb || pairs->y_len[p] > bb - yo)
        return m->fail(B2A_E_INVALID, "sequence offset/length outside seq_blob");
    }
    for (uint64_t p = 0; p < pairs->n_pairs; ++p)
      if (pairs->x_len[p] != pairs->y_len[p])
        return m->fail(B2A_E_INVALID, "pair " + std::to_string(p) +
                                          ": hamming distance cannot be calculated for texts of different length (" +
                                          std::to_string(pairs->x_len[p]) + "!=" + std::to_string(pairs->y_len[p]) + ")");
  }
  return run_split(
      m, pairs, nullptr, stats, false,
      [&](b2a_engine* e) { return b2a_hamming_batch(e, pairs, distance, status, stats); },
      [&](b2a_engine* e, const Share& s, b2a_stats* st) {
        return b2a_hamming_batch(e, &s.pairs, distance + s.lo, status ? status + s.lo : nullptr, st);
      });
}

}  // extern "C"

extern "C" {

int32_t b2a_multi_myers_batch(b2a_multi* m, const b2a_myers_match* match, uint32_t k, const b2a_pairs* pairs,
                              uint32_t* best_end, uint32_t* best_dist, uint64_t* n_hits, uint32_t* status,
                              b2a_stats* stats) {
  if (!m || !pairs || ((!best_end || !best_dist) && pairs->n_pairs)) return B2A_E_INVALID;
  if (!status && m->devs.size() > 1) {
    // an empty pattern fails the call; a share would name it by its index in the share, so the whole batch is
    // checked here first (offsets, then patterns, in the single engine's order) and the caller's index reported
    for (uint64_t p = 0; p < pairs->n_pairs; ++p) {
      const uint64_t bb = pairs->blob_bytes, xo = pairs->x_off[p], yo = pairs->y_off[p];
      if (xo > bb || pairs->x_len[p] > bb - xo || yo > bb || pairs->y_len[p] > bb - yo)
        return m->fail(B2A_E_INVALID, "sequence offset/length outside seq_blob");
    }
    for (uint64_t p = 0; p < pairs->n_pairs; ++p)
      if (pairs->x_len[p] == 0) return m->fail(B2A_E_INVALID, "pair " + std::to_string(p) + ": Pattern is empty");
  }
  const size_t nd = m->devs.size();
  std::vector<uint64_t> hits(nd, 0);
  std::vector<b2a_multi::HeldHits> held;
  const int32_t rc = run_split(
      m, pairs, nullptr, stats, false,
      [&](b2a_engine* e) {
        held = {{0, 0, pairs->n_pairs, 0}};
        return b2a_myers_batch(e, match, k, pairs, best_end, best_dist, n_hits ? &held[0].hits : nullptr, status,
                               stats);
      },
      [&](b2a_engine* e, const Share& s, b2a_stats* st) {
        const size_t d = (size_t)(std::find(m->eng.begin(), m->eng.end(), e) - m->eng.begin());
        return b2a_myers_batch(e, match, k, &s.pairs, best_end + s.lo, best_dist + s.lo, n_hits ? &hits[d] : nullptr,
                               status ? status + s.lo : nullptr, st);
      });
  if (rc || !n_hits) return rc;
  if (held.empty()) {  // the split ran: every entry holds its share
    const uint64_t per = (pairs->n_pairs + nd - 1) / nd;
    for (size_t d = 0; d < nd; ++d) {
      const uint64_t lo = std::min<uint64_t>(pairs->n_pairs, d * per);
      held.push_back({d, lo, std::min<uint64_t>(pairs->n_pairs, lo + per), hits[d]});
    }
  }
  *n_hits = 0;
  for (const auto& h : held) *n_hits += h.hits;
  m->myers_held = held;
  return B2A_OK;
}

int32_t b2a_multi_myers_hits_fetch(b2a_multi* m, uint64_t* hit_off, uint32_t* hit_end, uint32_t* hit_dist) {
  if (!m) return B2A_E_INVALID;
  if (m->myers_held.empty())
    return m->fail(B2A_E_STATE, "no hits are held: the last call was not b2a_multi_myers_batch with a listing");
  if (!hit_off) return B2A_E_INVALID;
  // one share after the other: a share's last offset is the next share's first, rewritten by it
  uint64_t base = 0;
  for (const auto& h : m->myers_held) {
    cudaSetDevice(m->devs[h.d]);
    const int32_t rc = b2a_myers_hits_fetch(m->eng[h.d], hit_off + h.lo, hit_end ? hit_end + base : nullptr,
                                            hit_dist ? hit_dist + base : nullptr);
    if (rc) return m->fail(rc, std::string("device ") + std::to_string(m->devs[h.d]) + ": " +
                                   b2a_last_error(m->eng[h.d]));
    for (uint64_t p = h.lo; p <= h.hi; ++p) hit_off[p] += base;
    base += h.hits;
  }
  return B2A_OK;
}

int32_t b2a_multi_pairhmm_batch(b2a_multi* m, const b2a_pairhmm_params* params, const b2a_pairs* pairs, double* prob,
                                uint32_t* status, b2a_stats* stats) {
  if (!m || !params || !pairs || (!prob && pairs->n_pairs)) return B2A_E_INVALID;
  const bool split = m->devs.size() > 1 && pairs->n_pairs >= m->devs.size();
  if (split && params->class_blob && params->n_classes >= 1 && params->n_classes < 256) {
    // a class byte out of range fails the call naming the pair; a share would name it by its index in the share, so
    // the whole batch is checked here first (offsets, then classes, in the single engine's order)
    for (uint64_t p = 0; p < pairs->n_pairs; ++p) {
      const uint64_t bb = pairs->blob_bytes, xo = pairs->x_off[p], yo = pairs->y_off[p];
      if (xo > bb || pairs->x_len[p] > bb - xo || yo > bb || pairs->y_len[p] > bb - yo)
        return m->fail(B2A_E_INVALID, "sequence offset/length outside seq_blob");
    }
    for (uint64_t p = 0; p < pairs->n_pairs; ++p) {
      const uint64_t off[2] = {pairs->x_off[p], pairs->y_off[p]};
      const uint32_t len[2] = {pairs->x_len[p], pairs->y_len[p]};
      for (int side = 0; side < 2; ++side)
        for (uint32_t i = 0; i < len[side]; ++i)
          if (params->class_blob[off[side] + i] >= params->n_classes)
            return m->fail(B2A_E_INVALID, "pair " + std::to_string(p) + ": class byte " +
                                              std::to_string(params->class_blob[off[side] + i]) + " >= n_classes (" +
                                              std::to_string(params->n_classes) + ")");
    }
  }
  if (!status && split) {
    // a NaN result fails the call naming the pair; a share would name it by its index in the share, so the shares run
    // with statuses and the caller's index of the first panic is reported here
    std::vector<uint32_t> st(pairs->n_pairs);
    const int32_t rc = b2a_multi_pairhmm_batch(m, params, pairs, prob, st.data(), stats);
    if (rc) return rc;
    for (uint64_t p = 0; p < pairs->n_pairs; ++p)
      if (st[p] != B2A_PAIR_OK) return m->fail(B2A_E_INVALID, "pair " + std::to_string(p) + ": assertion failed: !p.is_nan()");
    return B2A_OK;
  }
  return run_split(
      m, pairs, nullptr, stats, false,
      [&](b2a_engine* e) { return b2a_pairhmm_batch(e, params, pairs, prob, status, stats); },
      [&](b2a_engine* e, const Share& s, b2a_stats* st) {
        // the share's blob starts at its lowest offset: the class bytes move with it
        b2a_pairhmm_params ps = *params;
        if (ps.class_blob) ps.class_blob += s.pairs.seq_blob - pairs->seq_blob;
        return b2a_pairhmm_batch(e, &ps, &s.pairs, prob + s.lo, status ? status + s.lo : nullptr, st);
      });
}

}  // extern "C"
