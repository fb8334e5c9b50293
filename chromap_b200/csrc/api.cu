// chromap_b200 — C-ABI implementation (include/chromap_b200.h): context, device index / reference,
// batch pipeline driver (tiers, streams, events), stage entry points.  sm_90a.
#include <cuda_runtime.h>
#include <dlfcn.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <random>
#include <string>
#include <thread>
#include <tuple>
#include <type_traits>
#include <unordered_map>
#include <vector>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <thrust/iterator/transform_iterator.h>

#include "../../include/chromap_b200.h"
#include "cuda_owners.cuh"
#include "index_build.cuh"
#include "pipeline_kernels.cuh"
#include "seed_front.cuh"
#include "cta_pair_candidates.cuh"
#include "cta_verify_pairing.cuh"
#include "postprocess.cuh"
#include "allocate.cuh"
#include "exchange.cuh"
#include "sam_kernels.cuh"
#include "sam_text.cuh"
#include "ingest.cuh"
#include "lane_pipeline.cuh"
#include "host/read_range.h"

static_assert(sizeof(OutRecord) == sizeof(cmx_pe_record), "record layout");
static_assert(sizeof(cmx_pe_record) == 24, "record size");
static_assert(sizeof(OutPairs) == 24 && sizeof(cmx_pairs_record) == 24, "pairs record size");
static_assert(sizeof(OutSam) == sizeof(cmx_sam_record) && sizeof(OutSam) % 4 == 0 && SAM_MAX_CIGAR == CMX_SAM_MAX_CIGAR, "SAM record layout");

using DevBuf = DevMem<>;  // grow-only device buffer (ensure)

struct Tier {
  Caps caps;
  int slots_cap = 0;
  DevBuf mem;
  DevBuf ovf_list;   // pairs that overflowed THIS tier
  Scratch view{};
};

// Per-lane state of the batch pipeline.  A call that carries several whole reference batches is cut into up to
// CMX_MAX_LANES contiguous groups of batches; every group runs the full pipeline on its own stream (one host
// thread each), so the latency-bound kernels of one lane (overflow tiers, candidate pairing) share the SMs with
// the issue-bound kernels of another (minimizers, verification).
#define CMX_MAX_LANES 4
struct Lane {
  DevBuf rescue_list, verify_list, emit_list, nbest, sel, out_rec, out_n, offs, chunk_start, cub_tmp, bc_key, bc_ok, out_compact, bc_out;
  DevBuf bc2_list, bc2_over, bc2_slab;  // --bc-error-threshold 2 (DevWhitelist::c2_*)
  DevMem<Counters> ctr;
  DevMem<int> d_count;
  Tier tiers[N_TIERS];
  Stream stream, aux[N_TIERS - 1];  // aux: emit of the overflow tiers, beside tier 0's
  Event ev_join[N_TIERS - 1];
  // stage timing: a tier's start, front end done (tier 0), seeding, candidates, verification and pairing done; then the
  // start of selection, the start of emission and the compacted records
  Event ev_tier, ev_front, ev_seed, ev_pc, ev_ver, ev_pair, ev_select, ev_emit, ev_out;
  u32 p0 = 0, n = 0;  // pair range of the last call
  int tiers_used = 0;
  std::string err;
};

#define CMX_INGEST_SLOTS 6
struct IngestSlot {  // buffers of one cmx_ingest_fastq stream (text in, packed reads out)
  DevBuf text, nl, seq_start, qual_start, len, off, seq, qual, spans, tmp, stats, count, cut_stats;
  Stream stream;
};

struct cmx_ctx {
  int device = 0;
  cmx_params params;
  DevParams dp;
  std::string err;
  // reference
  DevMem<u8> ref_seq;
  DevMem<u64> ref_off;
  DevMem<u32> ref_len;
  u32 n_seq = 0;
  std::vector<u64> h_ref_off;
  std::vector<u32> h_ref_len;
  // index
  DevMem<ulonglong2> slots;
  u64 n_slots = 0;
  DevMem<u64> occ;
  u32 n_occ = 0;
  u64 n_keys = 0;
  int k = 0, w = 0;
  // scATAC barcode whitelist
  DevMem<ulonglong2> wl_slots;
  u64 wl_n_slots = 0, wl_num_sample = 0;
  DevMem<double> wl_pow;
  u32 wl_bc_len = 0;
  int wl_err = 1, wl_output_nw = 0, wl_active = 0;
  int wl_top_listed = 0;  // the key ~0 (all-T 32-mer) is listed with count wl_top_count: wl_lookup answers for it
  u64 wl_top_count = 0;
  double wl_prob = 0.9;
  DevBuf bc_seq, bc_qual;
  // --barcode-translate table (cmx_upload_barcode_translation); tr_n_slots == 0: none
  DevMem<ulonglong2> tr_slots;
  DevMem<char> tr_to;
  u64 tr_n_slots = 0;
  u32 tr_from_len = 0;
  // mapq tables
  DevMem<double> inv_log;
  DevMem<int> pen_thr;
  DevMem<u32> mt_init;  // std::mt19937(11) right after seeding
  // per-batch buffers
  DevBuf seq1, off1, seq2, off2, trace;
  Lane lanes[CMX_MAX_LANES];
  IngestSlot ingest[CMX_INGEST_SLOTS];
  int sf_grid = 132;            // persistent grid of the front-end kernel: SMs x resident CTAs (set by cmx_create)
  int n_lanes = CMX_MAX_LANES;  // lanes a multi-batch call is cut into (cmx_set_lanes; CMX_LANES overrides the default)
  int last_lanes_used = 0;
  Stream stream, up_stream, down_stream;
  // page-locked staging of h2d_big (allocated at the first big upload, kept: page-locking costs more than the copy)
  PinnedMem stage[2];
  Event stage_ev[2];
  Stream stage_stream;
  std::vector<Event> ev_up;
  Event ev_bc;
  Event ev[4];
  cmx_timing timing;
  u32 last_n_pairs = 0;
  // multi-GPU exchange (cmx_comm_init / cmx_dedup_exchange): an NCCL communicator of this context's own
  void *nccl_comm = nullptr;
  int comm_rank = 0, comm_size = 1;
};

static int fail(cmx_ctx *c, int code, const char *fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  if (c) c->err = buf;
  return code;
}
#define CU(call)                                                                                   \
  do {                                                                                             \
    cudaError_t e_ = (call);                                                                       \
    if (e_ != cudaSuccess) return fail(ctx, CMX_ERR_CUDA, "%s:%d %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_)); \
  } while (0)

static cudaError_t ensure(DevBuf &b, size_t bytes) { return bytes <= b.cap ? cudaSuccess : b.alloc(bytes + bytes / 8 + 256); }

// A kernel's dynamic shared-memory limit is one setting per process, shared by every context: it is only ever raised, so
// that a context sized for shorter reads never lowers it under one sized for longer reads.
template <typename K>
static cudaError_t raise_smem_limit(K *kernel, size_t bytes) {
  cudaFuncAttributes fa;
  cudaError_t e = cudaFuncGetAttributes(&fa, kernel);
  if (e == cudaSuccess && (size_t)fa.maxDynamicSharedSizeBytes < bytes) e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  return e;
}
// Everything sized by the longest read a context maps (cmx_create, cmx_set_max_read_length): the shared memory of the
// kernels that stage a whole read per thread or per tile or tier 0's hits per thread, the front end's persistent grid, and every lane's tier
// capacities.  The lanes' scratch must hold no tier laid out for other capacities (it is regrown from the new ones).
static cudaError_t size_for_read_length(cmx_ctx *ctx, int mrl) {
  cudaError_t e = cudaSuccess;
  if ((size_t)2 * mrl * 64 > 48 * 1024) e = raise_smem_limit(verify_kernel, (size_t)2 * mrl * 64);  // per-thread read-code columns (long reads)
  if (e == cudaSuccess) e = raise_smem_limit(cluster_kernel, (size_t)tier0_hits(mrl) * CLUSTER_NT * 8);  // tier 0's hit rows
  const size_t sf_smem = seed_front_smem_bytes(mrl);
  if (e == cudaSuccess) e = raise_smem_limit(seed_front_kernel<true>, sf_smem);
  if (e == cudaSuccess) e = raise_smem_limit(seed_front_kernel<false>, sf_smem);
  int per_sm = 0, n_sm = 0;
  if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, seed_front_kernel<true>, SF_NT, sf_smem);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, ctx->device);
  if (e != cudaSuccess) return e;
  ctx->sf_grid = std::max(1, per_sm) * std::max(1, n_sm);
  ctx->params.max_read_length = mrl;
  for (Lane &L : ctx->lanes)
    for (int t = 0; t < N_TIERS; ++t) L.tiers[t].caps = tier_caps(mrl, t);
  return cudaSuccess;
}
// the verification kernels' read-code columns (2 x 64 x max_read_length bytes of shared memory per CTA) bound the length
static const int MAX_READ_LENGTH_LIMIT = 1600;

extern "C" {

void cmx_default_params(cmx_params *p) {
  p->error_threshold = 8; p->min_num_seeds = 2; p->max_seed_freq0 = 500; p->max_seed_freq1 = 1000;
  p->max_num_best_mappings = 1; p->max_insert_size = 1000; p->mapq_threshold = 30; p->min_read_length = 30;
  p->drop_repetitive_reads = 500000; p->trim_adapters = 0; p->remove_pcr_duplicates = 0; p->tn5_shift = 0;
  p->split_alignment = 0; p->low_memory_mode = 0; p->output_format = 1; p->batch_size = 500000; p->max_read_length = 160;
  p->single_end = 0;
}

int cmx_apply_preset(cmx_params *p, const char *preset) {  // chromap_driver.cc:247-275
  const std::string s = preset ? preset : "";
  if (s.empty()) return CMX_OK;
  if (s == "atac") { p->max_insert_size = 2000; p->trim_adapters = 1; p->remove_pcr_duplicates = 1; p->tn5_shift = 1; p->low_memory_mode = 1; p->output_format = 1; return CMX_OK; }
  if (s == "chip") { p->max_insert_size = 2000; p->remove_pcr_duplicates = 1; p->low_memory_mode = 1; p->output_format = 1; return CMX_OK; }
  if (s == "hic") { p->error_threshold = 4; p->mapq_threshold = 1; p->split_alignment = 1; p->low_memory_mode = 1; p->output_format = 5; return CMX_OK; }
  return CMX_ERR_INVALID;
}

const char *cmx_last_error(const cmx_ctx *ctx) { return ctx ? ctx->err.c_str() : "null context"; }

int cmx_create(cmx_ctx **out, int device, const cmx_params *params) {
  if (!out || !params) return CMX_ERR_INVALID;
  *out = nullptr;
  int n_dev = 0;
  if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev <= 0 || device >= n_dev) return CMX_ERR_NO_DEVICE;
  if (!(((params->output_format == 1 || params->output_format == 2 || params->output_format == 4) && !params->split_alignment) ||
        (params->output_format == 5 && params->split_alignment)))
    return CMX_ERR_INVALID;  // BED / TagAlign (same records), SAM cores, or Hi-C pairs with split alignment
  if (params->output_format == 4 && (params->max_read_length > SAM_MAX_L_LONG || params->error_threshold > SAM_MAX_E)) return CMX_ERR_INVALID;
  if (params->error_threshold < 1 || params->error_threshold >= 16) return CMX_ERR_INVALID;  // mapping_parameters.h:80-88
  if (params->max_num_best_mappings < 1 || params->max_num_best_mappings > CMX_MAX_BEST) return CMX_ERR_INVALID;
  if (params->batch_size < 1 || params->max_read_length < params->min_read_length || params->max_read_length > MAX_READ_LENGTH_LIMIT) return CMX_ERR_INVALID;
  if (params->single_end && (params->split_alignment || params->output_format == 5)) return CMX_ERR_INVALID;  // single-end: BED / TagAlign only
  if (params->output_format == 5 && params->remove_pcr_duplicates && !params->low_memory_mode) return CMX_ERR_INVALID;  // pairs dedup: low-memory rule only
  std::unique_ptr<cmx_ctx> owner(new cmx_ctx);  // an early return deletes the partial context
  cmx_ctx *ctx = owner.get();
  ctx->device = device;
  ctx->params = *params;
  CU(cudaSetDevice(device));
  // The path's HBM traffic is random 16-byte table slots and short occurrence runs; CMX_L2_FETCH = 32 | 64 | 128 sets the L2
  // fetch-granularity hint for an A/B run (unset: the driver's default — the setting every committed number was measured with).
  if (const char *ev = getenv("CMX_L2_FETCH")) {
    const int gran = atoi(ev);
    if (gran == 32 || gran == 64 || gran == 128) { if (cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, (size_t)gran) != cudaSuccess) cudaGetLastError(); }
  }
  CU(ctx->stream.alloc()); CU(ctx->up_stream.alloc()); CU(ctx->down_stream.alloc());
  for (auto &e : ctx->ev) CU(e.alloc(cudaEventDefault));
  if (const char *ev = getenv("CMX_LANES")) ctx->n_lanes = std::max(1, std::min(CMX_MAX_LANES, atoi(ev)));
  for (Lane &L : ctx->lanes) {
    CU(L.stream.alloc());
    for (auto &a : L.aux) CU(a.alloc());
    for (auto &e : L.ev_join) CU(e.alloc(cudaEventDisableTiming));
    for (Event *e : {&L.ev_tier, &L.ev_front, &L.ev_seed, &L.ev_pc, &L.ev_ver, &L.ev_pair, &L.ev_select, &L.ev_emit, &L.ev_out}) CU(e->alloc(cudaEventDefault));
    CU(L.ctr.alloc(sizeof(Counters)));
    CU(L.d_count.alloc(sizeof(int) * 4));
  }
  {
    std::vector<double> il(65536, 0.0);
    std::vector<int> thr(96, 0x7fffffff);
    mapq_tables_fill(il.data(), thr.data());
    CU(ctx->inv_log.alloc(65536 * sizeof(double)));
    CU(ctx->pen_thr.alloc(96 * sizeof(int)));
    CU(cudaMemcpy(ctx->inv_log, il.data(), 65536 * sizeof(double), cudaMemcpyHostToDevice));
    CU(cudaMemcpy(ctx->pen_thr, thr.data(), 96 * sizeof(int), cudaMemcpyHostToDevice));
  }
  {
    std::vector<u32> mt(624);
    mt_init_fill(mt.data());
    CU(ctx->mt_init.alloc(624 * sizeof(u32)));
    CU(cudaMemcpy(ctx->mt_init, mt.data(), 624 * sizeof(u32), cudaMemcpyHostToDevice));
  }
  // the overflow-tier kernels may use more than the default 48 KB of (static + dynamic) shared memory
  CU(cudaFuncSetAttribute(cluster_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * CLUSTER_NT * 8));  // tier-0 hc = 64
  CU(cudaFuncSetAttribute(seed_cta_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
  CU(cudaFuncSetAttribute(pair_candidates_cta_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
  CU(cudaFuncSetAttribute(verify_cta_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
  CU(cudaFuncSetAttribute(pairing_cta_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
  CU(cudaFuncSetAttribute(verify_split_cta_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
  CU(size_for_read_length(ctx, params->max_read_length));
  memset(&ctx->timing, 0, sizeof(ctx->timing));
  *out = owner.release();
  return CMX_OK;
}

void cmx_destroy(cmx_ctx *ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);  // (the context's owners release on its device)
  cmx_comm_destroy(ctx);
  delete ctx;
}

// Pageable or file-mapped host memory -> device faster than one thread can copy it into the driver's staging area: eight
// threads fill one of two page-locked 32 MB buffers while cudaMemcpyAsync drains the other (a 3 Gbp index is 18 GB of
// arrays that the CLI hands over where they lie in the page cache).  Pinned or device sources go straight through.
static const size_t STAGE_BYTES = 32u << 20;
static cudaError_t h2d_big(cmx_ctx *ctx, void *dst, const void *src, size_t bytes) {
  if (bytes == 0) return cudaSuccess;
  cudaPointerAttributes at;
  const bool plain = cudaPointerGetAttributes(&at, src) == cudaSuccess && at.type == cudaMemoryTypeUnregistered;
  cudaGetLastError();
  if (!plain || bytes < STAGE_BYTES / 2) return cudaMemcpy(dst, src, bytes, cudaMemcpyDefault);
  if (!ctx->stage_stream) {
    if (ctx->stage[0].alloc(STAGE_BYTES) != cudaSuccess || ctx->stage[1].alloc(STAGE_BYTES) != cudaSuccess ||
        ctx->stage_ev[0].alloc(cudaEventDisableTiming) != cudaSuccess || ctx->stage_ev[1].alloc(cudaEventDisableTiming) != cudaSuccess ||
        ctx->stage_stream.alloc() != cudaSuccess) {  // (a failed alloc leaves the stream unset: the next big upload tries again)
      cudaGetLastError();
      return cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice);
    }
  }
  cudaStream_t st = ctx->stage_stream;
  cudaError_t rc = cudaSuccess;
  size_t i = 0;
  for (size_t o = 0; o < bytes && rc == cudaSuccess; o += STAGE_BYTES, ++i) {
    const int b = (int)(i & 1);
    const size_t n = std::min(STAGE_BYTES, bytes - o);
    if (i >= 2) rc = cudaEventSynchronize(ctx->stage_ev[b]);
    if (rc != cudaSuccess) break;
    const int nt = 8;
    const size_t slice = ((n + nt - 1) / nt + 4095) & ~(size_t)4095;
    char *stage = (char *)ctx->stage[b].h;
    std::thread th[8];
    for (int t = 0; t < nt; ++t)
      th[t] = std::thread([=]() {
        const size_t a = std::min(n, (size_t)t * slice), z = std::min(n, a + slice);
        if (z > a) memcpy(stage + a, (const char *)src + o + a, z - a);
      });
    for (int t = 0; t < nt; ++t) th[t].join();
    rc = cudaMemcpyAsync((char *)dst + o, stage, n, cudaMemcpyHostToDevice, st);
    if (rc == cudaSuccess) rc = cudaEventRecord(ctx->stage_ev[b], st);
  }
  const cudaError_t rs = cudaStreamSynchronize(st);
  return rc == cudaSuccess ? rs : rc;
}

int cmx_upload_reference(cmx_ctx *ctx, uint32_t n_seq, const uint64_t *offsets, const char *concat) {
  if (!ctx || !offsets || !concat || n_seq == 0) return CMX_ERR_INVALID;
  CU(cudaSetDevice(ctx->device));
  // the old reference goes before the new one is allocated; a failed upload leaves none
  ctx->ref_seq.reset(); ctx->ref_off.reset(); ctx->ref_len.reset();
  ctx->n_seq = 0; ctx->h_ref_off.clear(); ctx->h_ref_len.clear();
  std::vector<u64> doff(n_seq);
  std::vector<u32> dlen(n_seq);
  for (u32 i = 0; i < n_seq; ++i) {
    const u64 len = offsets[i + 1] - offsets[i];
    if (len >= 0xFFFFFFFFull) return fail(ctx, CMX_ERR_INVALID, "reference sequence %u too long for 32-bit positions", i);
    dlen[i] = (u32)len;
  }
  const u64 ref_bytes = ref_layout(n_seq, (const u64 *)offsets, doff.data());
  DevMem<u8> seq;
  DevMem<u64> d_off;
  DevMem<u32> d_len;
  CU(seq.alloc(ref_bytes));
  CU(cudaMemset(seq, 0, ref_bytes));
  CU(cudaDeviceSynchronize());  // (the staged copies below run on their own stream)
  for (u32 i = 0; i < n_seq; ++i)
    CU(h2d_big(ctx, seq + doff[i], concat + offsets[i], dlen[i]));  // host or device source
  CU(d_off.alloc(n_seq * sizeof(u64)));
  CU(d_len.alloc(n_seq * sizeof(u32)));
  CU(cudaMemcpy(d_off, doff.data(), n_seq * sizeof(u64), cudaMemcpyHostToDevice));
  CU(cudaMemcpy(d_len, dlen.data(), n_seq * sizeof(u32), cudaMemcpyHostToDevice));
  ctx->ref_seq = std::move(seq); ctx->ref_off = std::move(d_off); ctx->ref_len = std::move(d_len);
  ctx->n_seq = n_seq; ctx->h_ref_off = doff; ctx->h_ref_len = dlen;
  return CMX_OK;
}

static int table_shift(u64 n_slots) { int lg = 0; while ((1ull << lg) < n_slots) ++lg; return 64 - lg; }

// The mate-guided lookup (cta_pair_candidates.cuh) relies on every occurrence list holding distinct reference positions
// (true for any index Index::Construct builds: one k-mer per position).  Adjacent equal positions would break it: refuse.
__global__ void occ_check_kernel(const u64 *occ, u32 n, unsigned long long *bad) {
  const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i + 1 < n && (occ[i] >> 1) == (occ[i + 1] >> 1)) atomicAdd(bad, 1ull);
}
static int check_occurrences(cmx_ctx *ctx, const u64 *occ, u32 n_occ) {
  if (n_occ < 2) return CMX_OK;
  DevMem<unsigned long long> d_bad;
  unsigned long long bad = 0;
  CU(d_bad.alloc(8));
  CU(cudaMemset(d_bad, 0, 8));
  occ_check_kernel<<<(n_occ + 255) / 256, 256>>>(occ, n_occ, d_bad);
  CU(cudaMemcpy(&bad, d_bad, 8, cudaMemcpyDeviceToHost));
  if (bad) return fail(ctx, CMX_ERR_INVALID, "index: %llu adjacent occurrence entries share a reference position (not an index Chromap builds)", bad);
  return CMX_OK;
}

int cmx_upload_index(cmx_ctx *ctx, int k, int w, uint32_t n_buckets, const uint32_t *flags, const uint64_t *keys,
                     const uint64_t *vals, const uint64_t *occ, uint32_t n_occ) {
  if (!ctx || !flags || !keys || !vals || (n_occ && !occ)) return CMX_ERR_INVALID;
  if (k < 2 || k > 28 || w < 1 || w > CMX_W_MAX) return fail(ctx, CMX_ERR_INVALID, "unsupported k=%d w=%d", k, w);
  CU(cudaSetDevice(ctx->device));
  // occupied buckets (khash.h:165: 2 flag bits per bucket: 10 empty, 01 deleted, 00 occupied) are counted and inserted on
  // the device, straight from the reference's arrays: no host-side compaction pass over a billion buckets
  const u64 nbk = n_buckets;
  const size_t nfw = (size_t)((nbk + 15) / 16);
  DevMem<u32> d_flags;
  DevMem<unsigned long long> d_cnt;
  DevMem<u64> d_k, d_v;
  CU(d_flags.alloc(nfw * 4)); CU(d_cnt.alloc(8));
  CU(h2d_big(ctx, d_flags, flags, nfw * 4));
  CU(cudaMemset(d_cnt, 0, 8));
  khash_count_kernel<<<(unsigned)((nfw + 255) / 256), 256>>>(d_flags, nbk, d_cnt);
  unsigned long long n_keys = 0;
  CU(cudaMemcpy(&n_keys, d_cnt, 8, cudaMemcpyDeviceToHost));
  // the old index goes before the new table is allocated (a 3 Gbp table does not fit twice); a failed upload leaves none
  ctx->slots.reset(); ctx->occ.reset();
  ctx->n_slots = ctx->n_keys = 0; ctx->n_occ = 0; ctx->k = ctx->w = 0;
  u64 n_slots = 1024;  // load <= 0.5
  while (n_slots < 2 * n_keys) n_slots <<= 1;
  DevMem<ulonglong2> slots;
  CU(slots.alloc(n_slots * sizeof(ulonglong2)));
  CU(cudaMemset(slots, 0xFF, n_slots * sizeof(ulonglong2)));
  const size_t CH = 1u << 25;  // buckets per chunk: 2 x 256 MB in flight
  CU(d_k.alloc(std::min<size_t>(nbk, CH) * 8 + 16)); CU(d_v.alloc(std::min<size_t>(nbk, CH) * 8 + 16));
  for (u64 b0 = 0; b0 < nbk; b0 += CH) {
    const u64 n = std::min<u64>(CH, nbk - b0);
    CU(cudaStreamSynchronize(0));  // the previous chunk's insert kernel is done with d_k / d_v (the staged copies run on their own stream)
    CU(h2d_big(ctx, d_k, keys + b0, n * 8));
    CU(h2d_big(ctx, d_v, vals + b0, n * 8));
    khash_insert_kernel<<<(unsigned)((n + 255) / 256), 256>>>(d_flags, d_k, d_v, b0, n, slots, n_slots - 1, table_shift(n_slots));
    CU(cudaGetLastError());
  }
  CU(cudaDeviceSynchronize());
  d_flags.reset(); d_cnt.reset(); d_k.reset(); d_v.reset();
  DevMem<u64> d_occ;
  CU(d_occ.alloc((size_t)std::max<u32>(n_occ, 1) * sizeof(u64)));
  if (n_occ) CU(h2d_big(ctx, d_occ, occ, (size_t)n_occ * sizeof(u64)));
  const int rc = check_occurrences(ctx, d_occ, n_occ);
  if (rc) return rc;
  ctx->slots = std::move(slots); ctx->n_slots = n_slots; ctx->occ = std::move(d_occ); ctx->n_occ = n_occ; ctx->n_keys = n_keys;
  ctx->k = k; ctx->w = w;
  return CMX_OK;
}

int cmx_upload_barcode_whitelist(cmx_ctx *ctx, const uint64_t *keys, const uint32_t *counts, uint64_t n, uint64_t num_sample, uint32_t bc_len,
                                 int err_threshold, double prob_threshold, int output_not_in_whitelist) {
  if (!ctx || (n && (!keys || !counts)) || bc_len == 0 || bc_len > 32) return CMX_ERR_INVALID;
  if (err_threshold < 0 || err_threshold > 2)
    return fail(ctx, CMX_ERR_INVALID, "--bc-error-threshold %d: 0, 1 or 2 (a barcode is corrected by at most two substitutions; above 2 the extra Ns would stay in the key as A)", err_threshold);
  CU(cudaSetDevice(ctx->device));
  // the old whitelist goes before the new one is allocated; a failed upload leaves none
  ctx->wl_slots.reset(); ctx->wl_n_slots = 0; ctx->wl_active = 0;
  int top_listed = 0;
  u64 top_count = 0;
  for (u64 i = 0; i < n; ++i)
    if (keys[i] == CMX_EMPTY_KEY) { top_listed = 1; top_count = counts[i]; }
  u64 ns = 64;
  while (ns < 2 * n) ns <<= 1;
  DevMem<ulonglong2> slots;
  CU(slots.alloc(ns * sizeof(ulonglong2)));
  CU(cudaMemset(slots, 0xFF, ns * sizeof(ulonglong2)));
  if (n) {
    DevMem<u64> dk;
    DevMem<u32> dc;
    CU(dk.alloc(n * 8)); CU(dc.alloc(n * 4));
    CU(cudaMemcpy(dk, keys, n * 8, cudaMemcpyHostToDevice)); CU(cudaMemcpy(dc, counts, n * 4, cudaMemcpyHostToDevice));
    wl_insert_kernel<<<(unsigned)((n + 255) / 256), 256>>>(dk, dc, n, slots, ns - 1, table_shift(ns));
    CU(cudaGetLastError());
    CU(cudaDeviceSynchronize());
  }
  if (!ctx->wl_pow) {
    std::vector<double> pw(81);  // q of one base (3..40), or of two (6..80)
    for (int q = 0; q <= 80; ++q) pw[q] = pow(10.0, ((-q) / 10.0));  // host libm, chromap.cc:629-630, 681-682
    DevMem<double> d_pow;
    CU(d_pow.alloc(81 * sizeof(double)));
    CU(cudaMemcpy(d_pow, pw.data(), 81 * sizeof(double), cudaMemcpyHostToDevice));
    ctx->wl_pow = std::move(d_pow);
  }
  ctx->wl_slots = std::move(slots); ctx->wl_n_slots = ns; ctx->wl_num_sample = num_sample; ctx->wl_bc_len = bc_len; ctx->wl_err = err_threshold; ctx->wl_prob = prob_threshold;
  ctx->wl_output_nw = output_not_in_whitelist; ctx->wl_top_listed = top_listed; ctx->wl_top_count = top_count; ctx->wl_active = 1;
  return CMX_OK;
}

int cmx_upload_barcode_translation(cmx_ctx *ctx, const cmx_barcode_translation *t) {
  if (!ctx) return CMX_ERR_INVALID;
  if (t && (t->from_len < 1 || t->from_len > 31 || (t->n && (!t->keys || !t->to_off || (!t->to && t->to_off[t->n])))))
    return fail(ctx, CMX_ERR_INVALID, "barcode translation: FROM length %u (1..31) or missing arrays", t->from_len);
  CU(cudaSetDevice(ctx->device));
  // the old table goes before the new one is allocated; a failed upload leaves none
  ctx->tr_slots.reset(); ctx->tr_to.reset(); ctx->tr_n_slots = 0; ctx->tr_from_len = 0;
  if (!t) return CMX_OK;
  const u64 n = t->n;
  std::vector<u64> vals(n);
  for (u64 i = 0; i < n; ++i) {
    const u64 len = t->to_off[i + 1] - t->to_off[i];
    if (t->to_off[i + 1] < t->to_off[i] || len > 0xFFFFu || t->to_off[i] >> 48) return fail(ctx, CMX_ERR_INVALID, "barcode translation: TO string %llu out of range", (unsigned long long)i);
    vals[i] = t->to_off[i] << 16 | len;
  }
  u64 ns = 64;
  while (ns < 2 * n) ns <<= 1;
  DevMem<ulonglong2> slots;
  DevMem<char> to;
  CU(slots.alloc(ns * sizeof(ulonglong2)));
  CU(cudaMemset(slots, 0xFF, ns * sizeof(ulonglong2)));
  const u64 to_bytes = n ? t->to_off[n] : 0;
  CU(to.alloc(to_bytes + 1));
  if (to_bytes) CU(cudaMemcpy(to, t->to, to_bytes, cudaMemcpyHostToDevice));
  if (n) {
    DevMem<u64> dk, dv;
    CU(dk.alloc(n * 8)); CU(dv.alloc(n * 8));
    CU(cudaMemcpy(dk, t->keys, n * 8, cudaMemcpyHostToDevice)); CU(cudaMemcpy(dv, vals.data(), n * 8, cudaMemcpyHostToDevice));
    tr_insert_kernel<<<(unsigned)((n + 255) / 256), 256>>>(dk, dv, n, slots, ns - 1, table_shift(ns));
    CU(cudaGetLastError());
    CU(cudaDeviceSynchronize());
  }
  ctx->tr_slots = std::move(slots); ctx->tr_to = std::move(to); ctx->tr_n_slots = ns; ctx->tr_from_len = t->from_len;
  return CMX_OK;
}

int cmx_index_info(const cmx_ctx *ctx, int *k, int *w, uint64_t *n_keys, uint64_t *n_occ, uint64_t *table_slots) {
  if (!ctx || !ctx->slots) return CMX_ERR_STATE;
  if (k) *k = ctx->k;
  if (w) *w = ctx->w;
  if (n_keys) *n_keys = ctx->n_keys;
  if (n_occ) *n_occ = ctx->n_occ;
  if (table_slots) *table_slots = ctx->n_slots;
  return CMX_OK;
}

int cmx_build_index(cmx_ctx *ctx, int k, int w) {
  if (!ctx) return CMX_ERR_INVALID;
  if (!ctx->ref_seq) return fail(ctx, CMX_ERR_STATE, "upload the reference first");
  if (k < 2 || k > 28 || w < 1 || w > CMX_W_MAX) return fail(ctx, CMX_ERR_INVALID, "unsupported k=%d w=%d", k, w);
  CU(cudaSetDevice(ctx->device));
  IndexBuildResult r;
  std::string err;
  int rc = build_index_on_device(ctx->ref_seq, ctx->h_ref_off, ctx->h_ref_len, k, w, r, err);
  if (rc != 0) return fail(ctx, rc, "%s", err.c_str());
  rc = check_occurrences(ctx, r.occ, r.n_occ);
  if (rc) return rc;
  ctx->slots = std::move(r.slots); ctx->n_slots = r.n_slots; ctx->occ = std::move(r.occ); ctx->n_occ = r.n_occ; ctx->n_keys = r.n_keys;
  ctx->k = k; ctx->w = w;
  return CMX_OK;
}

// khash geometry + layout on the device: every (key, val) re-inserted with khash's own probe sequence
// (hash = key>>1 truncated to 32 bit, triangular steps; khash.h:232-245) so the reference's kh_get finds it.
__global__ void khash_layout_kernel(const ulonglong2 *slots, u64 n_slots, u64 *keys, u64 *vals, u32 mask) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_slots) return;
  const ulonglong2 kv = slots[i];
  if (kv.x == CMX_EMPTY_KEY) return;
  u32 b = (u32)(kv.x >> 1) & mask, step = 0;
  for (;;) {
    const u64 old = atomicCAS((unsigned long long *)&keys[b], (unsigned long long)CMX_EMPTY_KEY, (unsigned long long)kv.x);
    if (old == CMX_EMPTY_KEY) { vals[b] = kv.y; return; }
    b = (b + (++step)) & mask;
  }
}
__global__ void khash_flags_kernel(u64 *keys, u64 *vals, u32 n_buckets, u32 *flags) {
  const u32 wi = blockIdx.x * blockDim.x + threadIdx.x;  // one flag word = 16 buckets (khash.h:165)
  const u32 nf = n_buckets < 16 ? 1 : n_buckets >> 4;
  if (wi >= nf) return;
  u32 f = 0;
  for (u32 j = 0; j < 16; ++j) {
    const u32 b = wi * 16 + j;
    const bool empty = b >= n_buckets || keys[b] == CMX_EMPTY_KEY;
    if (empty) { f |= 2u << (j << 1); if (b < n_buckets) { keys[b] = 0; vals[b] = 0; } }
  }
  flags[wi] = f;
}

int cmx_download_index(cmx_ctx *ctx, uint32_t *n_buckets, uint32_t *n_keys, uint32_t *flags, uint64_t *keys, uint64_t *vals,
                       uint32_t *n_occ, uint64_t *occ) {
  if (!ctx || !ctx->slots) return CMX_ERR_STATE;
  CU(cudaSetDevice(ctx->device));
  // bucket count the reference's khash has after inserting n_keys keys (khash.h:295-300: it grows when
  // n_occupied >= upper_bound = n_buckets*0.77+0.5)
  u32 nb = 4;
  while ((u32)(nb * 0.77 + 0.5) < ctx->n_keys) nb <<= 1;
  if (n_buckets) *n_buckets = nb;
  if (n_keys) *n_keys = (u32)ctx->n_keys;
  if (n_occ) *n_occ = ctx->n_occ;
  if (occ && ctx->n_occ) CU(cudaMemcpy(occ, ctx->occ, (size_t)ctx->n_occ * sizeof(u64), cudaMemcpyDeviceToHost));
  if (flags && keys && vals) {
    const size_t nf = nb < 16 ? 1 : nb >> 4;
    DevMem<u64> dk, dv;
    DevMem<u32> df;
    CU(dk.alloc((size_t)nb * 8)); CU(dv.alloc((size_t)nb * 8)); CU(df.alloc(nf * 4));
    CU(cudaMemset(dk, 0xFF, (size_t)nb * 8)); CU(cudaMemset(dv, 0, (size_t)nb * 8));
    khash_layout_kernel<<<(unsigned)((ctx->n_slots + 255) / 256), 256>>>(ctx->slots, ctx->n_slots, dk, dv, nb - 1);
    khash_flags_kernel<<<(unsigned)((nf + 255) / 256), 256>>>(dk, dv, nb, df);
    CU(cudaGetLastError());
    CU(cudaDeviceSynchronize());
    CU(cudaMemcpy(keys, dk, (size_t)nb * 8, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(vals, dv, (size_t)nb * 8, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(flags, df, nf * 4, cudaMemcpyDeviceToHost));
  }
  return CMX_OK;
}

// ---------------------------------------------------------------------------------------------------
static cudaError_t tier_prepare(Tier &t, int n_slots, const int *pair_list, bool interleaved) {
  size_t o[SCRATCH_ARRAYS];
  if (n_slots > t.slots_cap) {
    const size_t want_slots = (size_t)n_slots + n_slots / 8 + 16;
    const size_t bytes = scratch_layout(t.caps, want_slots, interleaved, o);
    t.mem.reset();
    cudaError_t e = ensure(t.mem, bytes);
    if (e != cudaSuccess) return e;
    t.slots_cap = (int)want_slots;
  }
  scratch_layout(t.caps, t.slots_cap, interleaved, o);
  char *a[SCRATCH_ARRAYS];
  for (int i = 0; i < SCRATCH_ARRAYS; ++i) a[i] = (char *)t.mem.p + o[i];
  Scratch &S = t.view;
  S.caps = t.caps; S.n_slots = n_slots; S.pair_list = pair_list; S.mm_il = interleaved ? 1 : 0;
  scratch_bind(S, a);
  return cudaSuccess;
}

static int upload_batch(cmx_ctx *ctx, const cmx_batch *in, DevBatch *B) {
  const u32 n = in->n_pairs;
  if (in->on_device) {
    B->seq1 = (const u8 *)in->seq1; B->off1 = in->off1; B->seq2 = (const u8 *)in->seq2; B->off2 = in->off2;
  } else {
    const size_t b1 = in->off1[n], b2 = in->off2[n];
    CU(ensure(ctx->seq1, b1 + 64)); CU(ensure(ctx->seq2, b2 + 64));
    CU(ensure(ctx->off1, (n + 1) * 4)); CU(ensure(ctx->off2, (n + 1) * 4));
    CU(cudaMemcpyAsync(ctx->seq1.p, in->seq1, b1, cudaMemcpyHostToDevice, ctx->stream));
    CU(cudaMemcpyAsync(ctx->seq2.p, in->seq2, b2, cudaMemcpyHostToDevice, ctx->stream));
    CU(cudaMemcpyAsync(ctx->off1.p, in->off1, (n + 1) * 4, cudaMemcpyHostToDevice, ctx->stream));
    CU(cudaMemcpyAsync(ctx->off2.p, in->off2, (n + 1) * 4, cudaMemcpyHostToDevice, ctx->stream));
    B->seq1 = (const u8 *)ctx->seq1.p; B->off1 = (const u32 *)ctx->off1.p;
    B->seq2 = (const u8 *)ctx->seq2.p; B->off2 = (const u32 *)ctx->off2.p;
  }
  B->n_pairs = n; B->first_read_id = in->first_read_id; B->bc_ok = nullptr;
  return CMX_OK;
}

struct BatchAcc {  // per-call accumulators over sub-batches
  float ms_seed = 0, ms_pc = 0, ms_ver = 0, ms_pair = 0, ms_minimizer = 0, ms_cluster = 0, ms_select = 0, ms_emit = 0;
  u64 launches = 0, n_overflow = 0;
  Counters c;
  u64 tier_pairs[N_TIERS] = {0, 0, 0};
  int tiers_used = 0;
  BatchAcc() { memset(&c, 0, sizeof(c)); }
};

struct LaneJob {  // what one lane maps in one call: pairs [p0, p0 + n) of the call's batch
  u32 p0 = 0, n = 0;
  u32 piece = 0, piece0 = 0;                       // reads arrive in pieces of `piece` pairs; this lane's first piece index
  const std::vector<Event> *piece_ready = nullptr;
  const u8 *bc_seq = nullptr, *bc_qual = nullptr;  // device, already offset to p0
  u32 bc_len = 0;
  cudaEvent_t bc_ready = nullptr;
  bool want_bc = false;
  OutRecord *dst = nullptr;                        // device: compacted records of this lane (nullptr = lane buffer)
  u64 total = 0;
  BatchAcc acc;
  int rc = CMX_OK;
};

}  // extern "C"

// run_lane's side of the lane's launch sequence (lane_pipeline.cuh): kernels on the lane's stream, the overflow tiers' emits
// on its auxiliary streams, timing marks as events, list buffers grown on demand.  Like CUE, the first failing runtime call
// leaves its place and message in the lane's error; LANE_CU then makes no further runtime call and no kernel is launched.
#define LANE_CU(call) (!failed && ok((call), __LINE__, #call))
struct LaneOnDevice {
  Lane &L;
  const LaneJob &J;
  BatchAcc &acc;
  cudaStream_t s;
  u64 launches = 0;
  bool failed = false;
  bool ok(cudaError_t e, int line, const char *call) {
    if (e == cudaSuccess) return true;
    char b[512];
    snprintf(b, sizeof(b), "%s:%d %s: %s", __FILE__, line, call, cudaGetErrorString(e));
    L.err = b;
    failed = true;
    return false;
  }
  template <typename... KA, typename... A>
  void operator()(void (*kernel)(KA...), int grid, int block, size_t smem, A... a) {
    if (!failed) { kernel<<<grid, block, smem, s>>>(a...); ++launches; }
  }
  void mark(int m) {
    const cudaEvent_t ev[] = {L.ev_tier, L.ev_front, L.ev_seed, L.ev_pc, L.ev_ver, L.ev_pair, L.ev_select, L.ev_emit};
    LANE_CU(cudaEventRecord(ev[m], s));
  }
  void wait_piece(u32 q) { if (J.piece_ready) LANE_CU(cudaStreamWaitEvent(s, (*J.piece_ready)[J.piece0 + q], 0)); }
  Scratch tier(int t, int n, const int *pair_list) { LANE_CU(tier_prepare(L.tiers[t], n, pair_list, t == 0)); return L.tiers[t].view; }
  void *list(int l, size_t bytes) {
    DevBuf &b = l == LIST_RESCUE ? L.rescue_list : l == LIST_VERIFY ? L.verify_list : l == LIST_EMIT ? L.emit_list : L.tiers[l - LIST_OVERFLOW].ovf_list;
    LANE_CU(ensure(b, bytes));
    return b.p;
  }
  void clear_counts(int i, int n) { LANE_CU(cudaMemsetAsync(L.d_count + i, 0, n * sizeof(int), s)); }
  // waits for tier t; its stage times are taken here, before the next tier records the same events again
  int overflow_count(int t) {
    int n_ovf = 0;
    if (!LANE_CU(cudaMemcpyAsync(&n_ovf, L.d_count, sizeof(int), cudaMemcpyDeviceToHost, s)) || !LANE_CU(cudaStreamSynchronize(s)) || !LANE_CU(cudaGetLastError()))
      return 0;
    float f;
    cudaEventElapsedTime(&f, L.ev_tier, L.ev_seed); acc.ms_seed += f;
    if (t == 0) { cudaEventElapsedTime(&f, L.ev_tier, L.ev_front); acc.ms_minimizer += f; cudaEventElapsedTime(&f, L.ev_front, L.ev_seed); acc.ms_cluster += f; }
    cudaEventElapsedTime(&f, L.ev_seed, L.ev_pc); acc.ms_pc += f;
    cudaEventElapsedTime(&f, L.ev_pc, L.ev_ver); acc.ms_ver += f;
    cudaEventElapsedTime(&f, L.ev_ver, L.ev_pair); acc.ms_pair += f;
    return n_ovf;
  }
  const int *sort_list(int *list, int n) {
    std::vector<int> h(n);
    if (LANE_CU(cudaMemcpyAsync(h.data(), list, (size_t)n * 4, cudaMemcpyDeviceToHost, s)) && LANE_CU(cudaStreamSynchronize(s))) {
      std::sort(h.begin(), h.end());
      if (LANE_CU(cudaMemcpyAsync(list, h.data(), (size_t)n * 4, cudaMemcpyHostToDevice, s))) LANE_CU(cudaStreamSynchronize(s));
    }
    return list;
  }
  const int *chunk_starts(const std::vector<int> &c) {
    if (LANE_CU(ensure(L.chunk_start, c.size() * 4))) LANE_CU(cudaMemcpyAsync(L.chunk_start.p, c.data(), c.size() * 4, cudaMemcpyHostToDevice, s));
    return (const int *)L.chunk_start.p;
  }
  void emit_on(int t) {  // the overflow tiers' emits start on their own streams once the selection is done
    s = t == 0 ? L.stream.h : L.aux[t - 1].h;
    if (t > 0) LANE_CU(cudaStreamWaitEvent(s, L.ev_emit, 0));
  }
  void emit_join(int tiers_used) {
    s = L.stream;
    for (int t = 1; t < tiers_used; ++t)
      if (LANE_CU(cudaEventRecord(L.ev_join[t - 1], L.aux[t - 1]))) LANE_CU(cudaStreamWaitEvent(s, L.ev_join[t - 1], 0));
  }
};
#undef LANE_CU

// The uploaded whitelist as the barcode kernels see it, with lane L's correction lists for n barcodes at --bc-error-threshold 2.
static cudaError_t dev_whitelist(const cmx_ctx *ctx, Lane &L, u32 n, DevWhitelist *W) {
  W->slots = ctx->wl_slots; W->mask = ctx->wl_n_slots ? ctx->wl_n_slots - 1 : 0; W->shift = ctx->wl_n_slots ? table_shift(ctx->wl_n_slots) : 0;
  W->num_sample = (double)ctx->wl_num_sample; W->pow_tab = ctx->wl_pow; W->err_threshold = ctx->wl_err; W->prob_threshold = ctx->wl_prob;
  W->output_not_in_whitelist = ctx->wl_output_nw; W->active = ctx->wl_active; W->top_listed = ctx->wl_top_listed; W->top_count = ctx->wl_top_count;
  W->c2_list = W->c2_over = nullptr; W->c2_slab = nullptr;
  if (!ctx->wl_active || ctx->wl_err != 2) return cudaSuccess;
  cudaError_t e = ensure(L.bc2_list, (size_t)n * 4);
  if (e == cudaSuccess) e = ensure(L.bc2_over, (size_t)n * 4);
  if (e == cudaSuccess) e = ensure(L.bc2_slab, BC2_SLAB_WARPS * sizeof(Bc2Slab));
  W->c2_list = (u32 *)L.bc2_list.p; W->c2_over = (u32 *)L.bc2_over.p; W->c2_slab = (Bc2Slab *)L.bc2_slab.p;
  return e;
}

extern "C" {

// The whole device pipeline over pairs already resident in HBM (or landing piece by piece); records compacted in
// read order into the lane's buffer.  Synchronous on the lane's stream; safe to run one lane per host thread.
static int run_lane(cmx_ctx *ctx, Lane &L, const DevBatch &Bfull, LaneJob &J) {
  std::string &err = L.err;  // where CUE reports: lanes run on their own host threads and must not write ctx->err
  CUE(cudaSetDevice(ctx->device));
  const u32 n = J.n;
  BatchAcc &acc = J.acc;
  DevBatch B = Bfull;  // view of this lane's pairs: pair index i of the lane = pair p0 + i of the call
  B.off1 += J.p0; B.off2 += J.p0; B.n_pairs = n; B.first_read_id = Bfull.first_read_id + J.p0; B.bc_ok = nullptr;
  L.p0 = J.p0; L.n = n;
  const int mb = ctx->params.max_num_best_mappings;
  cudaStream_t st = L.stream;
  DevIndex ix;
  ix.slots = ctx->slots; ix.n_slots_mask = ctx->n_slots - 1; ix.shift = table_shift(ctx->n_slots); ix.occ = ctx->occ; ix.n_occ = ctx->n_occ; ix.k = ctx->k; ix.w = ctx->w;
  DevRef R;
  R.seq = ctx->ref_seq; R.off = ctx->ref_off; R.len = ctx->ref_len; R.n_seq = ctx->n_seq;
  MapqTables T;
  T.inv_log = ctx->inv_log; T.pen_thr = ctx->pen_thr;
  CUE(ensure(L.nbest, (size_t)n * 4)); CUE(ensure(L.sel, (size_t)n * mb * 4));
  const bool sam = ctx->params.output_format == 4;
  const size_t rec_bytes = sam ? sizeof(OutSam) : sizeof(OutRecord);
  CUE(ensure(L.out_rec, (size_t)n * mb * rec_bytes)); CUE(ensure(L.out_n, (size_t)(n + 1) * 4));
  CUE(ensure(L.offs, (size_t)(n + 1) * 8));
  OutRecord *dst = J.dst;
  if (!dst) { CUE(ensure(L.out_compact, (size_t)n * mb * rec_bytes)); dst = (OutRecord *)L.out_compact.p; }
  J.dst = dst;
  u64 *bc_dst = nullptr;
  if (J.want_bc && J.bc_seq) { CUE(ensure(L.bc_out, (size_t)n * mb * 8)); bc_dst = (u64 *)L.bc_out.p; }
  CUE(cudaMemsetAsync(L.nbest.p, 0, (size_t)n * 4, st));
  CUE(cudaMemsetAsync(L.out_n.p, 0, (size_t)(n + 1) * 4, st));
  CUE(cudaMemsetAsync(L.ctr, 0, sizeof(Counters), st));
  LaneOnDevice x{L, J, acc, st};
  if (J.bc_seq) {  // the barcode gate, when barcodes came with the batch
    DevWhitelist W;
    CUE(dev_whitelist(ctx, L, n, &W));
    CUE(ensure(L.bc_key, (size_t)n * 8)); CUE(ensure(L.bc_ok, (size_t)n));
    if (J.bc_ready) CUE(cudaStreamWaitEvent(st, J.bc_ready, 0));
    lane_barcodes(x, W, J.bc_seq, J.bc_qual, (int)J.bc_len, (int)n, (u64 *)L.bc_key.p, (u8 *)L.bc_ok.p, L.ctr.p);
    B.bc_ok = (const u8 *)L.bc_ok.p;
  }
  const LaneArgs a{dev_params(ctx->params, ctx->k, ctx->w), ix, R, B, T, ctx->mt_init, L.ctr, L.d_count, (int *)L.nbest.p, (int *)L.sel.p, (int *)L.out_n.p, L.out_rec.p, sam,
                   ctx->params.max_read_length};
  const LaneTiers tiers = lane_tiers(x, a, lane_front(x, a, J.piece_ready ? J.piece : n, ctx->sf_grid));
  lane_emit(x, a, tiers, (u32)ctx->params.batch_size);
  if (x.failed) return CMX_ERR_CUDA;
  // read-order compaction
  size_t tmp_bytes = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, (const int *)L.out_n.p, (u64 *)L.offs.p, (int)n + 1, st);
  CUE(ensure(L.cub_tmp, tmp_bytes));
  // out_n has n entries plus one trailing zero so that offs[n] = total
  cub::DeviceScan::ExclusiveSum(L.cub_tmp.p, tmp_bytes, (const int *)L.out_n.p, (u64 *)L.offs.p, (int)n + 1, st);
  const int cg = (int)((n + 255) / 256);
  if (sam) x(compact_words_kernel, cg, 256, 0, (int)n, mb, (int)(rec_bytes / 4), (const u32 *)L.out_rec.p, (const int *)L.out_n.p, (const u64 *)L.offs.p, (u32 *)dst);
  else x(compact_kernel, cg, 256, 0, (int)n, mb, (const OutRecord *)L.out_rec.p, (const int *)L.out_n.p, (const u64 *)L.offs.p, dst);
  if (bc_dst) x(compact_bc_kernel, cg, 256, 0, (int)n, (const int *)L.out_n.p, (const u64 *)L.offs.p, (const u64 *)L.bc_key.p, bc_dst);
  acc.launches += x.launches + 1;  // + the scan
  u64 total = 0;
  CUE(cudaEventRecord(L.ev_out, st));
  CUE(cudaMemcpyAsync(&total, (u64 *)L.offs.p + n, 8, cudaMemcpyDeviceToHost, st));
  Counters hc;
  CUE(cudaMemcpyAsync(&hc, L.ctr, sizeof(Counters), cudaMemcpyDeviceToHost, st));
  CUE(cudaStreamSynchronize(st));
  CUE(cudaGetLastError());
  float f;
  cudaEventElapsedTime(&f, L.ev_select, L.ev_emit); acc.ms_select += f;
  cudaEventElapsedTime(&f, L.ev_emit, L.ev_out); acc.ms_emit += f;
  {
    u64 *c = (u64 *)&acc.c;
    const u64 *b = (const u64 *)&hc;
    for (size_t i = 0; i < sizeof(Counters) / 8; ++i) c[i] += b[i];
  }
  for (int t = 0; t < tiers.used; ++t) acc.tier_pairs[t] += (u64)tiers.S[t].n_slots;
  acc.tiers_used = std::max(acc.tiers_used, tiers.used);
  acc.n_overflow += (u64)tiers.n_left + (sam ? hc.n_overflow : 0);  // SAM: reads / CIGARs beyond the fixed record
  J.total = total;
  L.tiers_used = tiers.used;
  return CMX_OK;
}

int cmx_map_batch_pe(cmx_ctx *ctx, const cmx_batch *in, cmx_records *out, void *user_stream) {
  if (!ctx || !in || !out) return CMX_ERR_INVALID;
  if (!ctx->slots || !ctx->ref_seq) return fail(ctx, CMX_ERR_STATE, "index and reference must be uploaded first");
  const u32 n = in->n_pairs;
  const int mb = ctx->params.max_num_best_mappings;
  out->n_records = 0; out->n_mapped_pairs = out->n_uniquely_mapped_pairs = out->n_candidates = out->n_overflow_pairs = 0;
  out->n_barcodes_in_whitelist = out->n_barcodes_corrected = 0;
  if (in->bc_seq && (in->bc_len == 0 || in->bc_len > 32 || !in->bc_qual)) return fail(ctx, CMX_ERR_INVALID, "barcodes need bc_qual and 1 <= bc_len <= 32");
  if (in->bc_seq && ctx->params.split_alignment) return fail(ctx, CMX_ERR_INVALID, "barcodes are not supported with split alignment");
  const bool se = ctx->params.single_end != 0;
  if (!in->seq1 || !in->off1 || (!se && (!in->seq2 || !in->off2))) return fail(ctx, CMX_ERR_INVALID, "cmx_batch: read pointers missing");
  if (n == 0) return CMX_OK;
  if (out->capacity < (u64)n * mb) return fail(ctx, CMX_ERR_INVALID, "records capacity %llu < n_pairs*max_num_best_mappings", (unsigned long long)out->capacity);
  CU(cudaSetDevice(ctx->device));
  (void)user_stream;  // the context's own streams are used; the call is synchronous
  cudaStream_t up = ctx->up_stream;
  const u32 bs = (u32)ctx->params.batch_size;
  const u32 n_sub = (n + bs - 1) / bs;  // reference batches in this call
  const bool bc = in->bc_seq && in->bc_len;
  CU(cudaEventRecord(ctx->ev[0], up));
  // ---- inputs: device pointers as they are; host buffers go up in pieces (one per reference batch) on the upload
  // stream, so the first kernels start on piece 0 while the other pieces are still in flight
  DevBatch B{};
  B.n_pairs = n; B.first_read_id = in->first_read_id;
  const u8 *bcs = nullptr, *bcq = nullptr;
  const bool pieces = !in->on_device;
  // upload granularity: a quarter of a reference batch, so the first kernels start after a sixteenth of a 4-batch upload
  const u32 ps = (bs % 4 == 0 && bs / 4 >= 32768) ? bs / 4 : bs;
  u32 n_pieces = 0;
  if (in->on_device) {
    B.seq1 = (const u8 *)in->seq1; B.off1 = in->off1; B.seq2 = (const u8 *)in->seq2; B.off2 = in->off2;
    if (bc) { bcs = (const u8 *)in->bc_seq; bcq = (const u8 *)in->bc_qual; }
  } else {
    const size_t b1 = in->off1[n], b2 = se ? 0 : in->off2[n];
    CU(ensure(ctx->seq1, b1 + 64)); CU(ensure(ctx->seq2, b2 + 64));
    CU(ensure(ctx->off1, (size_t)(n + 1) * 4)); CU(ensure(ctx->off2, (size_t)(n + 1) * 4));
    n_pieces = (n + ps - 1) / ps;
    while (ctx->ev_up.size() < n_pieces) { Event e; CU(e.alloc(cudaEventDisableTiming)); ctx->ev_up.push_back(std::move(e)); }
    CU(cudaMemcpyAsync(ctx->off1.p, in->off1, (size_t)(n + 1) * 4, cudaMemcpyHostToDevice, up));
    if (!se) CU(cudaMemcpyAsync(ctx->off2.p, in->off2, (size_t)(n + 1) * 4, cudaMemcpyHostToDevice, up));
    if (bc) {
      CU(ensure(ctx->bc_seq, (size_t)n * in->bc_len + 16)); CU(ensure(ctx->bc_qual, (size_t)n * in->bc_len + 16));
      CU(cudaMemcpyAsync(ctx->bc_seq.p, in->bc_seq, (size_t)n * in->bc_len, cudaMemcpyHostToDevice, up));
      CU(cudaMemcpyAsync(ctx->bc_qual.p, in->bc_qual, (size_t)n * in->bc_len, cudaMemcpyHostToDevice, up));
      if (!ctx->ev_bc) CU(ctx->ev_bc.alloc(cudaEventDisableTiming));
      CU(cudaEventRecord(ctx->ev_bc, up));
      bcs = (const u8 *)ctx->bc_seq.p; bcq = (const u8 *)ctx->bc_qual.p;
    }
    for (u32 s = 0; s < n_pieces; ++s) {
      const u32 p0 = s * ps, p1 = std::min(n, p0 + ps);
      CU(cudaMemcpyAsync((char *)ctx->seq1.p + in->off1[p0], in->seq1 + in->off1[p0], in->off1[p1] - in->off1[p0], cudaMemcpyHostToDevice, up));
      if (!se) CU(cudaMemcpyAsync((char *)ctx->seq2.p + in->off2[p0], in->seq2 + in->off2[p0], in->off2[p1] - in->off2[p0], cudaMemcpyHostToDevice, up));
      CU(cudaEventRecord(ctx->ev_up[s], up));
    }
    B.seq1 = (const u8 *)ctx->seq1.p; B.off1 = (const u32 *)ctx->off1.p;
    B.seq2 = (const u8 *)ctx->seq2.p; B.off2 = (const u32 *)ctx->off2.p;
  }
  CU(cudaEventRecord(ctx->ev[1], up));
  // ---- lanes: contiguous groups of whole reference batches (the sampling generator restarts per batch chunk,
  // so a lane needs nothing from its neighbours)
  const int n_lanes = (int)std::min<u32>((u32)ctx->n_lanes, n_sub);
  LaneJob jobs[CMX_MAX_LANES];
  for (int l = 0; l < n_lanes; ++l) {
    const u32 s0 = (u32)((u64)n_sub * l / n_lanes), s1 = (u32)((u64)n_sub * (l + 1) / n_lanes);
    LaneJob &J = jobs[l];
    J.p0 = s0 * bs; J.n = std::min(n, s1 * bs) - J.p0;
    if (pieces) { J.piece = ps; J.piece0 = s0 * (bs / ps); J.piece_ready = &ctx->ev_up; }
    if (bc) { J.bc_seq = bcs + (size_t)J.p0 * in->bc_len; J.bc_qual = bcq + (size_t)J.p0 * in->bc_len; J.bc_len = in->bc_len; J.bc_ready = pieces ? ctx->ev_bc.h : nullptr; }
    J.want_bc = bc && out->barcode_keys;
    if (out->on_device && n_lanes == 1) J.dst = (OutRecord *)out->records;
  }
  // every lane maps its pairs and then delivers its records itself, behind the records of the lanes before it (their
  // counts are known as soon as those lanes have finished mapping), so the copies of early lanes overlap later lanes
  std::atomic<int> mapped[CMX_MAX_LANES];
  for (auto &f : mapped) f.store(0);
  const size_t rec_bytes = ctx->params.output_format == 4 ? sizeof(OutSam) : sizeof(OutRecord);
  auto lane_main = [&](int l) {
    LaneJob &J = jobs[l];
    Lane &L = ctx->lanes[l];
    J.rc = run_lane(ctx, L, B, J);
    if (J.rc) J.total = 0;
    mapped[l].store(1, std::memory_order_release);
    u64 before = 0;
    for (int k = 0; k < l; ++k) {
      while (!mapped[k].load(std::memory_order_acquire)) std::this_thread::yield();
      before += jobs[k].total;
    }
    if (J.rc || !J.total) return;
    cudaError_t e = cudaSuccess;
    if ((void *)J.dst != (void *)out->records)
      e = cudaMemcpyAsync((char *)out->records + before * rec_bytes, J.dst, J.total * rec_bytes, out->on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, L.stream);
    if (e == cudaSuccess && J.want_bc) e = cudaMemcpyAsync(out->barcode_keys + before, L.bc_out.p, J.total * 8, cudaMemcpyDeviceToHost, L.stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(L.stream);
    if (e != cudaSuccess) { L.err = std::string("record copy: ") + cudaGetErrorString(e); J.rc = CMX_ERR_CUDA; }
  };
  CU(cudaEventRecord(ctx->ev[2], ctx->down_stream));
  {
    std::vector<std::thread> th;
    for (int l = 1; l < n_lanes; ++l) th.emplace_back(lane_main, l);
    lane_main(0);
    for (auto &t : th) t.join();
  }
  CU(cudaEventRecord(ctx->ev[3], ctx->down_stream));
  CU(cudaStreamSynchronize(ctx->down_stream));
  ctx->last_lanes_used = n_lanes;
  ctx->last_n_pairs = n;
  for (int l = 0; l < n_lanes; ++l)
    if (jobs[l].rc) { ctx->err = ctx->lanes[l].err; return jobs[l].rc; }
  u64 total = 0;
  for (int l = 0; l < n_lanes; ++l) total += jobs[l].total;
  CU(cudaGetLastError());
  float ms_h2d = 0, ms_call = 0;
  cudaEventElapsedTime(&ms_h2d, ctx->ev[0], ctx->ev[1]);
  cudaEventElapsedTime(&ms_call, ctx->ev[2], ctx->ev[3]);  // lanes launched .. last record delivered (events on an idle stream)
  BatchAcc acc;
  for (int l = 0; l < n_lanes; ++l) {
    const BatchAcc &a = jobs[l].acc;
    acc.ms_seed += a.ms_seed; acc.ms_pc += a.ms_pc; acc.ms_ver += a.ms_ver; acc.ms_pair += a.ms_pair; acc.ms_minimizer += a.ms_minimizer;
    acc.ms_cluster += a.ms_cluster; acc.ms_select += a.ms_select; acc.ms_emit += a.ms_emit;
    acc.launches += a.launches; acc.n_overflow += a.n_overflow;
    u64 *x = (u64 *)&acc.c;
    const u64 *y = (const u64 *)&a.c;
    for (size_t i = 0; i < sizeof(Counters) / 8; ++i) x[i] += y[i];
    for (int t = 0; t < N_TIERS; ++t) acc.tier_pairs[t] += a.tier_pairs[t];
  }
  out->n_records = total;
  out->n_mapped_pairs = acc.c.n_mapped; out->n_uniquely_mapped_pairs = acc.c.n_unique; out->n_candidates = acc.c.n_candidates;
  out->n_overflow_pairs = acc.n_overflow;
  out->n_barcodes_in_whitelist = acc.c.n_bc_in_whitelist; out->n_barcodes_corrected = acc.c.n_bc_corrected;
  cmx_timing &tm = ctx->timing;
  memset(&tm, 0, sizeof(tm));
  // stage times are sums over the lanes' own streams; lanes overlap, so they add up to more than total_ms
  tm.h2d_ms = ms_h2d; tm.d2h_ms = 0;  // record copies run on the lanes' own streams, overlapped with other lanes' kernels
  tm.seed_ms = acc.ms_seed; tm.front_ms = acc.ms_minimizer; tm.reserved_ms = 0; tm.cluster_ms = acc.ms_cluster;
  tm.pair_candidates_ms = acc.ms_pc; tm.verify_ms = acc.ms_ver; tm.pairing_ms = acc.ms_pair; tm.select_ms = acc.ms_select; tm.emit_ms = acc.ms_emit;
  tm.total_ms = ms_call;
  tm.n_minimizers = acc.c.n_minimizers; tm.n_probe_steps = acc.c.n_probe_steps; tm.n_found = acc.c.n_found; tm.n_occ_reads = acc.c.n_occ_reads;
  tm.n_verified = acc.c.n_verified; tm.n_launches = acc.launches;
  for (int t = 0; t < 3; ++t) tm.tier_pairs[t] = acc.tier_pairs[t];
  for (int r = 0; r < 8; ++r) tm.escalations[r] = acc.c.ovf_reason[r];
  if (acc.n_overflow) return fail(ctx, CMX_ERR_OVERFLOW, "%llu pair(s) exceeded the largest scratch tier", (unsigned long long)acc.n_overflow);
  return CMX_OK;
}

// Host helper: bytes taken by the first min(max_records, complete) 4-line records of `text` (a record is complete when
// its fourth newline is present).
uint64_t cmx_fastq_cut(const char *text, uint64_t n_bytes, uint32_t max_records, uint32_t *n_records) {
  uint64_t pos = 0, end_of_last = 0;
  uint32_t lines = 0, recs = 0;
  while (recs < max_records) {
    const void *q = memchr(text + pos, '\n', n_bytes - pos);
    if (!q) break;
    pos = (uint64_t)((const char *)q - text) + 1;
    if (++lines == 4) { lines = 0; ++recs; end_of_last = pos; }
  }
  if (n_records) *n_records = recs;
  return end_of_last;
}

int cmx_ingest_fastq(cmx_ctx *ctx, int slot, const char *text, uint64_t n_bytes, int want_qual, uint32_t *name_spans, cmx_ingested *out) {
  return cmx_ingest_fastq_range(ctx, slot, text, n_bytes, want_qual, name_spans, nullptr, out);
}

int cmx_ingest_fastq_range(cmx_ctx *ctx, int slot, const char *text, uint64_t n_bytes, int want_qual, uint32_t *name_spans, const cmx_read_range *range,
                           cmx_ingested *out) {
  if (!ctx || !out || slot < 0 || slot >= CMX_INGEST_SLOTS || (!text && n_bytes)) return CMX_ERR_INVALID;
  if (range && !cmxhost::ReadRangeRepresentable(*range)) return fail(ctx, CMX_ERR_INVALID, "cmx_ingest_fastq_range: a read range that is not representable");
  const bool cut = range && !cmxhost::ReadRangeIsWhole(*range);
  static_assert(CUT_MAX_RANGES == CMX_MAX_READ_RANGES, "range count");
  CutRanges cr{};
  if (cut) {
    cr.n = range->n; cr.reverse = range->reverse;
    for (u32 k = 0; k < range->n; ++k) { cr.start[k] = range->start[k]; cr.end[k] = range->end[k]; }
  }
  memset(out, 0, sizeof(*out));
  if (n_bytes == 0) return CMX_OK;
  if (n_bytes >= 0xFFFFFFF0ull) return fail(ctx, CMX_ERR_INVALID, "cmx_ingest_fastq: chunk of 4 GiB or more");
  if (text[n_bytes - 1] != '\n') return fail(ctx, CMX_ERR_INVALID, "cmx_ingest_fastq: the chunk must end at a record boundary (cmx_fastq_cut)");
  CU(cudaSetDevice(ctx->device));
  IngestSlot &g = ctx->ingest[slot];
  if (!g.stream) CU(g.stream.alloc());
  cudaStream_t st = g.stream;
  const u32 nb = (u32)n_bytes;
  CU(ensure(g.text, n_bytes + 16)); CU(ensure(g.nl, ((size_t)nb + 16) * 4)); CU(ensure(g.count, 16)); CU(ensure(g.stats, sizeof(IngestStats)));
  CU(cudaMemcpyAsync(g.text.p, text, n_bytes, cudaMemcpyHostToDevice, st));
  // newline positions: select the indices whose byte is '\n'
  thrust::counting_iterator<u32> idx(0);
  CU(ensure(g.qual_start, (size_t)nb));  // newline flags live here until the per-record arrays are sized (same buffer, reused)
  u8 *flags = (u8 *)g.qual_start.p;
  newline_flag_kernel<<<(nb + 255) / 256, 256, 0, st>>>((const char *)g.text.p, nb, flags);
  size_t tb = 0;
  cub::DeviceSelect::Flagged(nullptr, tb, idx, flags, (u32 *)g.nl.p, (u32 *)g.count.p, (int)nb, st);
  CU(ensure(g.tmp, tb));
  CU(cub::DeviceSelect::Flagged(g.tmp.p, tb, idx, flags, (u32 *)g.nl.p, (u32 *)g.count.p, (int)nb, st));
  u32 n_nl = 0;
  CU(cudaMemcpyAsync(&n_nl, g.count.p, 4, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  if (n_nl % 4 != 0) return fail(ctx, CMX_ERR_INVALID, "cmx_ingest_fastq: %u lines is not a whole number of 4-line records", n_nl);
  const u32 n = n_nl / 4;
  CU(ensure(g.seq_start, (size_t)n * 4)); CU(ensure(g.qual_start, (size_t)n * 4)); CU(ensure(g.len, (size_t)(n + 1) * 4)); CU(ensure(g.off, (size_t)(n + 1) * 4));
  if (name_spans) CU(ensure(g.spans, (size_t)n * 8));
  IngestStats hs = {0, 0, 0, 0, 0xFFFFFFFFu, 0};
  CU(cudaMemcpyAsync(g.stats.p, &hs, sizeof(hs), cudaMemcpyHostToDevice, st));
  CU(cudaMemsetAsync((u32 *)g.len.p + n, 0, 4, st));
  ingest_record_kernel<<<(n + 255) / 256, 256, 0, st>>>((const char *)g.text.p, (const u32 *)g.nl.p, n, (u32 *)g.seq_start.p, (u32 *)g.qual_start.p, (u32 *)g.len.p,
                                                        name_spans ? (u32 *)g.spans.p : nullptr, (IngestStats *)g.stats.p);
  CutStats hc = {0, 0, 0xFFFFFFFFu, 0};
  if (cut) {
    CU(ensure(g.cut_stats, sizeof(CutStats)));
    CU(cudaMemcpyAsync(g.cut_stats.p, &hc, sizeof(hc), cudaMemcpyHostToDevice, st));
    ingest_cut_len_kernel<<<(n + 255) / 256, 256, 0, st>>>((u32 *)g.len.p, n, cr, (CutStats *)g.cut_stats.p);
  }
  cub::DeviceScan::ExclusiveSum(nullptr, tb, (const u32 *)g.len.p, (u32 *)g.off.p, (int)n + 1, st);
  CU(ensure(g.tmp, tb));
  CU(cub::DeviceScan::ExclusiveSum(g.tmp.p, tb, (const u32 *)g.len.p, (u32 *)g.off.p, (int)n + 1, st));
  // sequence bytes never exceed the chunk; a malformed record (quality shorter than sequence) is only reported after the
  // pack kernel has run, so the buffers are sized by the chunk and the quality copy is bounded by the quality line itself
  CU(ensure(g.seq, n_bytes + 64));
  if (want_qual) CU(ensure(g.qual, n_bytes + 64));
  // (a cut is never longer than its read: the same sizes hold)
  if (cut)
    ingest_cut_pack_kernel<<<(unsigned)(((u64)n * 32 + 255) / 256), 256, 0, st>>>((const char *)g.text.p, (const u32 *)g.seq_start.p, (const u32 *)g.qual_start.p,
                                                                                 (const u32 *)g.off.p, (const u32 *)g.nl.p, n, cr, (char *)g.seq.p,
                                                                                 want_qual ? (char *)g.qual.p : nullptr);
  else
    ingest_pack_kernel<<<(unsigned)(((u64)n * 32 + 255) / 256), 256, 0, st>>>((const char *)g.text.p, (const u32 *)g.seq_start.p, (const u32 *)g.qual_start.p,
                                                                             (const u32 *)g.off.p, (const u32 *)g.nl.p, n, (char *)g.seq.p, want_qual ? (char *)g.qual.p : nullptr);
  CU(cudaMemcpyAsync(&hs, g.stats.p, sizeof(hs), cudaMemcpyDeviceToHost, st));
  if (cut) CU(cudaMemcpyAsync(&hc, g.cut_stats.p, sizeof(hc), cudaMemcpyDeviceToHost, st));
  if (name_spans) CU(cudaMemcpyAsync(name_spans, g.spans.p, (size_t)n * 8, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  CU(cudaGetLastError());
  if (hs.bad_header || hs.bad_plus) return fail(ctx, CMX_ERR_INVALID, "cmx_ingest_fastq: not 4-line FASTQ (%u headers without '@', %u separator lines without '+')", hs.bad_header, hs.bad_plus);
  if (hs.empty_reads) return fail(ctx, CMX_ERR_INVALID, "cmx_ingest_fastq: %u empty reads (the reference skips them per file; use the host reader)", hs.empty_reads);
  if (hs.qual_mismatch) return fail(ctx, CMX_ERR_INVALID, "cmx_ingest_fastq: %u records whose quality and sequence lengths differ", hs.qual_mismatch);
  if (cut && (hc.out_of_range || hc.empty))
    return fail(ctx, CMX_ERR_READ_RANGE, "cmx_ingest_fastq_range: %u reads end before a range of the read format does, %u reads are empty after the cut", hc.out_of_range,
                hc.empty);
  if (cut) { hs.min_len = hc.min_len; hs.max_len = hc.max_len; }
  out->n_reads = n; out->seq = (const char *)g.seq.p; out->off = (const uint32_t *)g.off.p; out->qual = want_qual ? (const char *)g.qual.p : nullptr;
  out->min_len = n ? hs.min_len : 0; out->max_len = hs.max_len;
  return CMX_OK;
}

int cmx_host_register(void *ptr, uint64_t bytes) {
  if (!ptr || !bytes) return CMX_ERR_INVALID;
  return cudaHostRegister(ptr, (size_t)bytes, cudaHostRegisterPortable) == cudaSuccess ? CMX_OK : CMX_ERR_CUDA;
}
int cmx_host_unregister(void *ptr) {
  if (!ptr) return CMX_ERR_INVALID;
  return cudaHostUnregister(ptr) == cudaSuccess ? CMX_OK : CMX_ERR_CUDA;
}

int cmx_set_lanes(cmx_ctx *ctx, int n_lanes) {
  if (!ctx || n_lanes < 1 || n_lanes > CMX_MAX_LANES) return CMX_ERR_INVALID;
  if (n_lanes != ctx->n_lanes) {
    // each lane's tiers are sized for the pairs it last mapped: a 4-lane split of a 2 M-pair call and the 1-lane call that
    // follows it do not fit an 80 GB device together with a 3 Gbp index, so the old split's scratch goes first
    CU(cudaSetDevice(ctx->device));
    CU(cudaDeviceSynchronize());
    for (Lane &L : ctx->lanes)
      for (Tier &t : L.tiers) { t.mem.reset(); t.ovf_list.reset(); t.slots_cap = 0; }
  }
  ctx->n_lanes = n_lanes;
  return CMX_OK;
}

int cmx_set_max_read_length(cmx_ctx *ctx, int32_t L) {
  if (!ctx) return CMX_ERR_INVALID;
  const cmx_params &p = ctx->params;
  if (L < p.min_read_length || L > MAX_READ_LENGTH_LIMIT || (p.output_format == 4 && L > SAM_MAX_L_LONG))
    return fail(ctx, CMX_ERR_INVALID, "max_read_length %d: use %d .. %d%s", (int)L, p.min_read_length, p.output_format == 4 ? SAM_MAX_L_LONG : MAX_READ_LENGTH_LIMIT,
                p.output_format == 4 ? " with SAM output" : "");
  CU(cudaSetDevice(ctx->device));
  int smem_optin = 0;
  CU(cudaDeviceGetAttribute(&smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, ctx->device));
  if (seed_front_smem_bytes(L) > (size_t)smem_optin)  // 64 reads per front-end tile: up to 843 bases in an H100's 227 KB
    return fail(ctx, CMX_ERR_INVALID, "max_read_length %d: the front end's read tiles need %zu bytes of shared memory, the device has %d", (int)L,
                seed_front_smem_bytes(L), smem_optin);
  CU(cudaDeviceSynchronize());
  // every tier's scratch was laid out for the old capacities: released here, regrown by the next call (as cmx_set_lanes does)
  for (Lane &Ln : ctx->lanes)
    for (Tier &t : Ln.tiers) { t.mem.reset(); t.ovf_list.reset(); t.slots_cap = 0; }
  CU(size_for_read_length(ctx, L));
  return CMX_OK;
}

int cmx_last_batch_timing(cmx_ctx *ctx, cmx_timing *out) {
  if (!ctx || !out) return CMX_ERR_INVALID;
  *out = ctx->timing;
  return CMX_OK;
}

__global__ void trace_kernel(Scratch S, cmx_pair_trace *out, u32 p0) {
  const int slot = blockIdx.x * blockDim.x + threadIdx.x;
  if (slot >= S.n_slots) return;
  const PairMeta &pm = S.pmeta[slot];
  if (pm.status == ST_OVERFLOW) return;
  cmx_pair_trace t;
  memset(&t, 0, sizeof(t));
  const ReadMeta *rm = S.rmeta + 2 * slot;
  for (int m = 0; m < 2; ++m) {
    t.trimmed_len[m] = rm[m].len;
    t.n_minimizers[m] = rm[m].n_mm;
    t.n_pos_candidates_gen[m] = rm[m].n_cand_gen[0]; t.n_neg_candidates_gen[m] = rm[m].n_cand_gen[1];
    t.n_pos_candidates[m] = rm[m].n_cand[0]; t.n_neg_candidates[m] = rm[m].n_cand[1];
    t.n_pos_mappings[m] = rm[m].n_map[0]; t.n_neg_mappings[m] = rm[m].n_map[1];
    t.min_errors[m] = rm[m].min_err; t.second_min_errors[m] = rm[m].second_min_err;
    t.n_best[m] = rm[m].n_best; t.n_second_best[m] = rm[m].n_second_best;
    t.repetitive_seed_length[m] = rm[m].rep_len;
  }
  t.supplement_result = pm.sup;
  t.min_sum_errors = pm.min_sum; t.second_min_sum_errors = pm.second_min_sum; t.n_best_pairs = pm.n_best; t.n_second_best_pairs = pm.n_second_best;
  t.n_records = pm.n_rec;
  out[p0 + slot_pair(S, slot)] = t;
}

int cmx_last_batch_trace(cmx_ctx *ctx, cmx_pair_trace *out, uint32_t n_pairs) {
  if (!ctx || !out || n_pairs != ctx->last_n_pairs) return CMX_ERR_INVALID;
  CU(cudaSetDevice(ctx->device));
  CU(ensure(ctx->trace, (size_t)n_pairs * sizeof(cmx_pair_trace)));
  CU(cudaMemset(ctx->trace.p, 0, (size_t)n_pairs * sizeof(cmx_pair_trace)));
  for (int l = 0; l < ctx->last_lanes_used; ++l) {
    const Lane &L = ctx->lanes[l];
    for (int t = 0; t < L.tiers_used; ++t) {
      const Scratch S = L.tiers[t].view;
      trace_kernel<<<(S.n_slots + 255) / 256, 256>>>(S, (cmx_pair_trace *)ctx->trace.p, L.p0);
    }
  }
  CU(cudaDeviceSynchronize());
  CU(cudaMemcpy(out, ctx->trace.p, (size_t)n_pairs * sizeof(cmx_pair_trace), cudaMemcpyDeviceToHost));
  return CMX_OK;
}

// ---- stage entry points ---------------------------------------------------------------------------
__global__ void stage_minimizers_kernel(DevBatch B, int k, int w, u64 *out_hash, u32 *out_pos, int *out_n, u32 stride) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= 2 * (int)B.n_pairs) return;
  const int pair = r >> 1, mate = r & 1;
  const u8 *seq = read_ptr(B, pair, mate);
  u64 *oh = out_hash + (size_t)r * stride;
  u32 *op = out_pos + (size_t)r * stride;
  int n = 0;
  minimizer_scan_any([&](int i) { return seq[i]; }, read_raw_len(B, pair, mate), k, w, [&](u64 h, u32 p) { if (n < (int)stride) { oh[n] = h; op[n] = p; } ++n; });
  out_n[r] = n;
}

int cmx_stage_minimizers(cmx_ctx *ctx, const cmx_batch *in, uint64_t *out_hash, uint32_t *out_pos, int32_t *out_n, uint32_t stride) {
  if (!ctx || !in || !out_hash || !out_pos || !out_n) return CMX_ERR_INVALID;
  if (!ctx->k) return fail(ctx, CMX_ERR_STATE, "index (k, w) not set");
  CU(cudaSetDevice(ctx->device));
  DevBatch B{};
  int rc = upload_batch(ctx, in, &B);
  if (rc) return rc;
  const size_t R = 2 * (size_t)in->n_pairs;
  DevMem<u64> dh;
  DevMem<u32> dp;
  DevMem<int> dn;
  CU(dh.alloc(R * stride * 8)); CU(dp.alloc(R * stride * 4)); CU(dn.alloc(R * 4));
  stage_minimizers_kernel<<<(unsigned)((R + 127) / 128), 128, 0, ctx->stream>>>(B, ctx->k, ctx->w, dh, dp, dn, stride);
  CU(cudaStreamSynchronize(ctx->stream));
  CU(cudaGetLastError());
  CU(cudaMemcpy(out_hash, dh, R * stride * 8, cudaMemcpyDeviceToHost));
  CU(cudaMemcpy(out_pos, dp, R * stride * 4, cudaMemcpyDeviceToHost));
  CU(cudaMemcpy(out_n, dn, R * 4, cudaMemcpyDeviceToHost));
  return CMX_OK;
}

__global__ void stage_probe_kernel(DevIndex ix, const u64 *h, u64 n, u8 *found, u64 *key, u64 *val) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  u64 v = 0;
  int steps;
  const int kind = index_lookup(ix, h[i], &v, &steps);
  found[i] = kind != 0;
  key[i] = kind ? ((h[i] << 1) | (kind == 1 ? 1u : 0u)) : 0;
  val[i] = v;
}

int cmx_stage_probe(cmx_ctx *ctx, const uint64_t *hashes, uint64_t n, uint8_t *found, uint64_t *key, uint64_t *val) {
  if (!ctx || !hashes || !found || !key || !val) return CMX_ERR_INVALID;
  if (!ctx->slots) return fail(ctx, CMX_ERR_STATE, "index not uploaded");
  CU(cudaSetDevice(ctx->device));
  DevIndex ix;
  ix.slots = ctx->slots; ix.n_slots_mask = ctx->n_slots - 1; ix.shift = table_shift(ctx->n_slots); ix.occ = ctx->occ; ix.n_occ = ctx->n_occ; ix.k = ctx->k; ix.w = ctx->w;
  DevMem<u64> dh, dk, dv;
  DevMem<u8> df;
  CU(dh.alloc(n * 8 + 8)); CU(dk.alloc(n * 8 + 8)); CU(dv.alloc(n * 8 + 8)); CU(df.alloc(n + 8));
  CU(cudaMemcpy(dh, hashes, n * 8, cudaMemcpyHostToDevice));
  if (n) stage_probe_kernel<<<(unsigned)((n + 255) / 256), 256>>>(ix, dh, n, df, dk, dv);
  CU(cudaDeviceSynchronize());
  CU(cudaGetLastError());
  CU(cudaMemcpy(found, df, n, cudaMemcpyDeviceToHost)); CU(cudaMemcpy(key, dk, n * 8, cudaMemcpyDeviceToHost)); CU(cudaMemcpy(val, dv, n * 8, cudaMemcpyDeviceToHost));
  return CMX_OK;
}

}  // extern "C"
// The stage entries' side of a launch sequence of lane_pipeline.cuh: kernels on the legacy default stream.
struct StageLaunch {
  template <typename... KA, typename... A>
  void operator()(void (*kernel)(KA...), int grid, int block, size_t smem, A... a) { kernel<<<grid, block, smem>>>(a...); }
};
extern "C" {

int cmx_stage_correct_barcodes(cmx_ctx *ctx, const char *bc_seq, const char *bc_qual, uint64_t n, uint32_t bc_len, uint64_t *out_key, uint8_t *out_ok,
                               uint64_t *n_in_whitelist, uint64_t *n_corrected) {
  if (!ctx || (n && (!bc_seq || !bc_qual || !out_key || !out_ok)) || bc_len == 0 || bc_len > 32 || n > 0x7FFFFFFFull) return CMX_ERR_INVALID;
  if (!ctx->wl_active) return fail(ctx, CMX_ERR_STATE, "barcode whitelist not uploaded");
  if (bc_len != ctx->wl_bc_len) return fail(ctx, CMX_ERR_INVALID, "barcodes of %u bases, the whitelist's are %u", bc_len, ctx->wl_bc_len);
  CU(cudaSetDevice(ctx->device));
  Counters hc{};
  if (n) {
    DevMem<u8> ds, dq, dok;
    DevMem<u64> dkey;
    DevMem<Counters> dc;
    CU(ds.alloc(n * bc_len)); CU(dq.alloc(n * bc_len)); CU(dok.alloc(n)); CU(dkey.alloc(n * 8)); CU(dc.alloc(sizeof(Counters)));
    CU(cudaMemcpy(ds, bc_seq, n * bc_len, cudaMemcpyHostToDevice)); CU(cudaMemcpy(dq, bc_qual, n * bc_len, cudaMemcpyHostToDevice));
    CU(cudaMemset(dc, 0, sizeof(Counters)));
    DevWhitelist W;
    CU(dev_whitelist(ctx, ctx->lanes[0], (u32)n, &W));
    StageLaunch x;
    lane_barcodes(x, W, (const u8 *)ds.p, (const u8 *)dq.p, (int)bc_len, (int)n, (u64 *)dkey.p, (u8 *)dok.p, (Counters *)dc.p);
    CU(cudaGetLastError());
    CU(cudaDeviceSynchronize());
    CU(cudaMemcpy(out_key, dkey, n * 8, cudaMemcpyDeviceToHost)); CU(cudaMemcpy(out_ok, dok, n, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(&hc, dc, sizeof(Counters), cudaMemcpyDeviceToHost));
  }
  if (n_in_whitelist) *n_in_whitelist = hc.n_bc_in_whitelist;
  if (n_corrected) *n_corrected = hc.n_bc_corrected;
  return CMX_OK;
}

__global__ void stage_align_kernel(int e, int L, const u8 *pat, const u8 *txt, u64 n, int *err, int *endp) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const u8 *p = pat + i * (size_t)(L + 2 * e), *t = txt + i * (size_t)L;
  int ep = 0;
  err[i] = banded_align(e, L, [&](int j) { return base_code(p[j]); }, [&](int j) { return base_code(t[j]); }, &ep);
  endp[i] = ep;
}

int cmx_stage_banded_align(cmx_ctx *ctx, int e, int read_len, const char *patterns, const char *texts, uint64_t n, int32_t *num_errors, int32_t *end_pos) {
  if (!ctx || !patterns || !texts || !num_errors || !end_pos || e < 1 || e > 15 || read_len < 1) return CMX_ERR_INVALID;
  CU(cudaSetDevice(ctx->device));
  DevMem<u8> dp, dt;
  DevMem<int> de, dq;
  const size_t pb = n * (size_t)(read_len + 2 * e), tb = n * (size_t)read_len;
  CU(dp.alloc(pb + 8)); CU(dt.alloc(tb + 8)); CU(de.alloc(n * 4 + 8)); CU(dq.alloc(n * 4 + 8));
  CU(cudaMemcpy(dp, patterns, pb, cudaMemcpyHostToDevice)); CU(cudaMemcpy(dt, texts, tb, cudaMemcpyHostToDevice));
  if (n) stage_align_kernel<<<(unsigned)((n + 127) / 128), 128>>>(e, read_len, dp, dt, n, de, dq);
  CU(cudaDeviceSynchronize());
  CU(cudaGetLastError());
  CU(cudaMemcpy(num_errors, de, n * 4, cudaMemcpyDeviceToHost)); CU(cudaMemcpy(end_pos, dq, n * 4, cudaMemcpyDeviceToHost));
  return CMX_OK;
}

__global__ void __launch_bounds__(CTA_NT) stage_cta_sort_kernel(u64 *keys, u8 *tags, int n, int sm_cap, int with_tags) {
  extern __shared__ u64 smk_stage[];
  u8 *smt = (u8 *)(smk_stage + sm_cap);
  if (with_tags) {
    auto cless = [](u64 pa, u8 ca, u64 pb, u8 cb) { return ca != cb ? ca > cb : pa < pb; };  // candidate order
    cta_sort_pairs<u8>(keys, tags, n, ~0ull, (u8)0, cless, smk_stage, smt, sm_cap);
  } else {
    cta_sort_keys(keys, n, smk_stage, sm_cap);
  }
}

int cmx_stage_cta_sort(cmx_ctx *ctx, uint64_t *keys, uint8_t *tags, uint32_t n, uint32_t sm_cap) {
  if (!ctx || !keys || sm_cap < 2 || (sm_cap & (sm_cap - 1)) || sm_cap > CTA_SORT_SMEM_MAX) return CMX_ERR_INVALID;
  CU(cudaSetDevice(ctx->device));
  size_t cap = 1;
  while (cap < n) cap <<= 1;
  DevMem<u64> dk;
  DevMem<u8> dt;
  CU(dk.alloc(cap * 8 + 8)); CU(dt.alloc(cap + 8));
  CU(cudaMemcpy(dk, keys, (size_t)n * 8, cudaMemcpyHostToDevice));
  if (tags) CU(cudaMemcpy(dt, tags, n, cudaMemcpyHostToDevice));
  stage_cta_sort_kernel<<<1, CTA_NT, (size_t)sm_cap * 9>>>(dk, dt, (int)n, (int)sm_cap, tags ? 1 : 0);
  CU(cudaDeviceSynchronize());
  CU(cudaGetLastError());
  CU(cudaMemcpy(keys, dk, (size_t)n * 8, cudaMemcpyDeviceToHost));
  if (tags) CU(cudaMemcpy(tags, dt, n, cudaMemcpyDeviceToHost));
  return CMX_OK;
}

// ---- post-processing (host side of the writer; GPU sort is a later row) ----------------------------
static inline auto rec_key(const cmx_pe_record &r) {  // bed_mapping.h:208-215 prefixed by rid
  return std::make_tuple(r.rid, r.fragment_start, r.fragment_length, r.mapq, r.direction, r.is_unique, r.read_id,
                         r.positive_alignment_length, r.negative_alignment_length);
}
static inline void tn5(cmx_pe_record &r) {  // bed_mapping.h:225-230
  r.fragment_start += 4; r.positive_alignment_length -= 4; r.fragment_length -= 9; r.negative_alignment_length -= 5;
}
static inline void tn5_se(cmx_pe_record &r) {  // single-end, bed_mapping.h:97-103
  if (r.direction == 1) r.fragment_start += 4; else r.fragment_length -= 5;
}

// cmx_postprocess / cmx_postprocess_bc under given parameters (the allocation runs them twice with others than the context's)
static void postprocess_host(const cmx_params &p, cmx_pe_record *recs, uint64_t n, uint64_t *n_out);
static void postprocess_bc_host(const cmx_params &p, cmx_pe_record *recs, uint64_t *bcs, uint64_t n, uint64_t *n_out);
int cmx_postprocess(cmx_ctx *ctx, cmx_pe_record *recs, uint64_t n, uint64_t *n_out) {
  if (!ctx || (!recs && n) || !n_out) return CMX_ERR_INVALID;
  postprocess_host(ctx->params, recs, n, n_out);
  return CMX_OK;
}
static void postprocess_host(const cmx_params &p, cmx_pe_record *recs, uint64_t n, uint64_t *n_out) {
  *n_out = 0;
  if (n == 0) return;
  auto less = [](const cmx_pe_record &a, const cmx_pe_record &b) { return rec_key(a) < rec_key(b); };
  const bool se = p.single_end != 0;  // single-end duplicates: same start on the same sequence (bed_mapping.h:89-92)
  auto same = [se](const cmx_pe_record &a, const cmx_pe_record &b) {
    return a.rid == b.rid && a.fragment_start == b.fragment_start && (se || a.fragment_length == b.fragment_length);
  };
  auto tn5 = [se](cmx_pe_record &r) { if (se) tn5_se(r); else ::tn5(r); };
  uint64_t o = 0;
  if (p.low_memory_mode) {  // mapping_writer.h:166-376
    std::sort(recs, recs + n, less);
    uint64_t i = 0;
    while (i < n) {
      cmx_pe_record keep = recs[i];
      uint32_t dups = 1;
      uint64_t j = i + 1;
      if (p.remove_pcr_duplicates)
        for (; j < n && same(recs[j], recs[i]); ++j) { ++dups; if (recs[j].mapq > keep.mapq) keep = recs[j]; }
      if (keep.mapq >= p.mapq_threshold) {
        keep.num_dups = (uint8_t)std::min<uint32_t>(255, dups);
        if (p.tn5_shift) tn5(keep);
        recs[o++] = keep;
      }
      i = j;
    }
    *n_out = o;
    return;
  }
  if (p.tn5_shift) for (uint64_t i = 0; i < n; ++i) tn5(recs[i]);  // chromap.h:1322-1355
  std::sort(recs, recs + n, less);
  if (p.remove_pcr_duplicates) {  // mapping_processor.h:161-202: keeps the last of each run
    uint64_t i = 0, w = 0;
    while (i < n) {
      uint64_t j = i + 1;
      while (j < n && same(recs[j], recs[i])) ++j;
      cmx_pe_record keep = recs[j - 1];
      keep.num_dups = (uint8_t)std::min<uint64_t>(255, j - i);
      recs[w++] = keep;
      i = j;
    }
    n = w;
  }
  for (uint64_t i = 0; i < n; ++i) if (recs[i].mapq >= p.mapq_threshold) recs[o++] = recs[i];
  *n_out = o;
}

int cmx_postprocess_pairs(cmx_ctx *ctx, cmx_pairs_record *recs, uint64_t n, uint64_t *n_out) {
  if (!ctx || (!recs && n) || !n_out) return CMX_ERR_INVALID;
  const cmx_params &p = ctx->params;
  // records live in the bucket of rid1; the merge order is (bucket, PairsMapping::operator<) (pairs_mapping.h:40-43)
  std::sort(recs, recs + n, [](const cmx_pairs_record &a, const cmx_pairs_record &b) {
    return std::make_tuple(a.rid1, a.rid2, a.pos1, a.pos2, a.mapq, a.read_id) < std::make_tuple(b.rid1, b.rid2, b.pos1, b.pos2, b.mapq, b.read_id);
  });
  uint64_t o = 0;
  if (p.remove_pcr_duplicates) {  // mapping_writer.h:234-300 with PairsMapping::operator== (pairs_mapping.h:44-49)
    uint64_t i = 0;
    while (i < n) {
      cmx_pairs_record keep = recs[i];
      uint64_t j = i + 1;
      for (; j < n && recs[j].rid1 == recs[i].rid1 && recs[j].pos1 == recs[i].pos1 && recs[j].rid2 == recs[i].rid2 && recs[j].pos2 == recs[i].pos2; ++j)
        if (recs[j].mapq > keep.mapq) keep = recs[j];
      if (keep.mapq >= p.mapq_threshold) recs[o++] = keep;
      i = j;
    }
  } else {
    for (uint64_t i = 0; i < n; ++i) if (recs[i].mapq >= p.mapq_threshold) recs[o++] = recs[i];
  }
  *n_out = o;
  return CMX_OK;
}

int64_t cmx_format_pairs(const char *const *names, const uint32_t *lengths, uint32_t n_seq, const cmx_pairs_record *recs, uint64_t n,
                         const char *const *read_names, uint32_t first_read_id, char *buf, int64_t cap) {
  int64_t len = 0;
  std::string hdr = "## pairs format v1.0.0\n#shape: upper triangle\n";  // mapping_writer.cc:383-402
  for (uint32_t i = 0; i < n_seq; ++i) hdr += std::string("#chromsize: ") + names[i] + " " + std::to_string(lengths[i]) + "\n";
  hdr += "#columns: readID chrom1 pos1 chrom2 pos2 strand1 strand2 pair_type mapq1 mapq2\n";
  if (buf && (int64_t)hdr.size() <= cap) memcpy(buf, hdr.data(), hdr.size());
  len += (int64_t)hdr.size();
  for (uint64_t i = 0; i < n; ++i) {  // mapping_writer.cc:405-421
    const cmx_pairs_record &r = recs[i];
    const std::string line = std::string(read_names[r.read_id - first_read_id]) + "\t" + names[r.rid1] + "\t" + std::to_string(r.pos1 + 1) + "\t" + names[r.rid2] +
                             "\t" + std::to_string(r.pos2 + 1) + "\t" + (r.strand1 ? "+" : "-") + "\t" + (r.strand2 ? "+" : "-") + "\tUU\t" +
                             std::to_string(r.mapq) + "\t" + std::to_string(r.mapq) + "\n";
    if (buf && len + (int64_t)line.size() <= cap) memcpy(buf + len, line.data(), line.size());
    len += (int64_t)line.size();
  }
  return len;
}

int cmx_postprocess_bc(cmx_ctx *ctx, cmx_pe_record *recs, uint64_t *bcs, uint64_t n, uint64_t *n_out) {
  if (!ctx || (n && (!recs || !bcs)) || !n_out) return CMX_ERR_INVALID;
  postprocess_bc_host(ctx->params, recs, bcs, n, n_out);
  return CMX_OK;
}
static void postprocess_bc_host(const cmx_params &p, cmx_pe_record *recs, uint64_t *bcs, uint64_t n, uint64_t *n_out) {
  *n_out = 0;
  if (n == 0) return;
  std::vector<cmx_pe_record> rr(recs, recs + n);
  std::vector<uint64_t> bb(bcs, bcs + n);
  if (!p.low_memory_mode && p.tn5_shift) for (auto &r : rr) { if (p.single_end) tn5_se(r); else tn5(r); }
  std::vector<uint64_t> ord(n);
  for (uint64_t i = 0; i < n; ++i) ord[i] = i;
  auto key = [&](uint64_t i) {  // bed_mapping.h:145-153 prefixed by rid
    const cmx_pe_record &r = rr[i];
    return std::make_tuple(r.rid, r.fragment_start, r.fragment_length, bb[i], r.mapq, r.direction, r.is_unique, r.read_id);
  };
  std::sort(ord.begin(), ord.end(), [&](uint64_t a, uint64_t b) { return key(a) < key(b); });
  const bool se = p.single_end != 0;
  auto same = [&](uint64_t a, uint64_t b) {  // cell-level duplicates: bed_mapping.h:154-159 (paired-end), :36-39 (single-end: barcode + start)
    return rr[a].rid == rr[b].rid && rr[a].fragment_start == rr[b].fragment_start && (se || rr[a].fragment_length == rr[b].fragment_length) && bb[a] == bb[b];
  };
  uint64_t o = 0, i = 0;
  while (i < n) {
    uint64_t j = i + 1, keep = ord[i];
    uint32_t dups = 1;
    if (p.remove_pcr_duplicates)
      for (; j < n && same(ord[j], ord[j - 1]); ++j) {  // consecutive equality (single-end: the key is not a prefix of the order)
        ++dups;
        if (p.low_memory_mode) { if (rr[ord[j]].mapq > rr[keep].mapq) keep = ord[j]; }
        else keep = ord[j];
      }
    cmx_pe_record k = rr[keep];
    if (k.mapq >= p.mapq_threshold) {
      if (p.remove_pcr_duplicates) k.num_dups = (uint8_t)std::min<uint32_t>(255, dups);
      if (p.low_memory_mode && p.tn5_shift) { if (se) tn5_se(k); else tn5(k); }
      recs[o] = k; bcs[o] = bb[keep]; ++o;
    }
    i = j;
  }
  *n_out = o;
}

int64_t cmx_format_bed_bc(const char *const *names, const cmx_pe_record *recs, const uint64_t *bcs, uint64_t n, uint32_t bc_len, char *buf, int64_t cap) {
  int64_t len = 0;
  static const char tab[4] = {'A', 'C', 'G', 'T'};
  for (uint64_t i = 0; i < n; ++i) {  // mapping_writer.cc:127-137, barcode_translator.h:114-123
    const cmx_pe_record &r = recs[i];
    std::string line = std::string(names[r.rid]) + "\t" + std::to_string(r.fragment_start) + "\t" + std::to_string((uint32_t)(r.fragment_start + r.fragment_length)) + "\t";
    for (uint32_t j = 0; j < bc_len; ++j) line.push_back(tab[(bcs[i] >> ((bc_len - 1 - j) * 2)) & 3]);
    line += "\t" + std::to_string((uint32_t)r.num_dups) + "\n";
    if (buf && len + (int64_t)line.size() <= cap) memcpy(buf + len, line.data(), line.size());
    len += (int64_t)line.size();
  }
  return len;
}

// Sort + duplicate removal + MAPQ filter (+ Tn5 shift) over device-resident records: d_a[0, n) (and d_bca) in, the result in
// d_b[0, *nsel) (and d_bcb); d_a is used as scratch.  All four buffers hold n entries.  Work is queued on ctx->stream and
// waited for.
struct MaxU64 {
  __device__ u64 operator()(u64 a, u64 b) const { return a > b ? a : b; }
};
static size_t pp_bulk_tmp_bytes(u64 n, cudaStream_t st) {  // CUB scratch of pp_bulk_resolve
  size_t a = 0, b = 0;
  cub::DeviceScan::InclusiveSum(nullptr, a, (const u32 *)nullptr, (u32 *)nullptr, (int)n, st);
  cub::DeviceReduce::ReduceByKey(nullptr, b, (const u32 *)nullptr, (u32 *)nullptr, (const u64 *)nullptr, (u64 *)nullptr, (u32 *)nullptr, MaxU64(), (int)n, st);
  return std::max(a, b);
}
// Bulk-level duplicate removal (postprocess.cuh, pp_bulk_*) of the sorted barcoded records recs / bcs [0, n): one candidate per
// bulk group in res / res_bc [0, *n_groups), keep_flag set by the MAPQ filter.  k0, k1 (n u64), i0, i1 (n u32) and tmp
// (pp_bulk_tmp_bytes) are scratch.  CMX_ERR_INVALID for a barcode that is not in the whitelist.
static int pp_bulk_resolve(cmx_ctx *ctx, const PpParams &P, const PpAbundance &wl, const PpRecord *recs, const u64 *bcs, u64 n, u64 *k0, u64 *k1, u32 *i0, u32 *i1,
                           DevMem<> &tmp, PpRecord *res, u64 *res_bc, u8 *keep_flag, u64 *n_groups_out) {
  cudaStream_t st = ctx->stream;
  const unsigned nb = (unsigned)((n + 255) / 256);
  DevMem<u32> d_small;  // [0] groups, [1] highest MAPQ of the last group, [2..3] barcodes missing from the whitelist (u64)
  CU(d_small.alloc(16));
  CU(cudaMemsetAsync(d_small, 0, 16, st));
  PpAbundance A = wl;
  A.n_missing = (unsigned long long *)(d_small.p + 2);
  pp_bulk_entry_kernel<<<nb, 256, 0, st>>>(P.se, recs, bcs, n, A, i0, k0);
  size_t tmp_bytes = tmp.cap;
  CU(cub::DeviceScan::InclusiveSum(tmp.p, tmp_bytes, i0, i1, (int)n, st));  // i1 = 1-based group of each record
  tmp_bytes = tmp.cap;
  CU(cub::DeviceReduce::ReduceByKey(tmp.p, tmp_bytes, i1, i0, k0, k1, d_small.p, MaxU64(), (int)n, st));  // k1[g] = best key of group g
  u32 small[4] = {0, 0, 0, 0};
  CU(cudaMemcpyAsync(small, d_small, 16, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  CU(cudaGetLastError());
  const u32 n_groups = small[0];
  const u64 n_missing = (u64)small[2] | ((u64)small[3] << 32);
  if (n_missing)
    return fail(ctx, CMX_ERR_INVALID, "bulk-level duplicate removal: %llu barcode(s) of the records are not in the whitelist, whose abundance the rule needs",
                (unsigned long long)n_missing);
  pp_bulk_heads_kernel<<<nb, 256, 0, st>>>(i1, n, i0);  // i0[g] = first record of group g
  pp_bulk_last_mapq_kernel<<<nb, 256, 0, st>>>(recs, i0, n_groups, n, d_small.p + 1);
  pp_bulk_resolve_kernel<<<(n_groups + 255) / 256, 256, 0, st>>>(P, recs, bcs, k1, i0, n_groups, n, d_small.p + 1, res, res_bc, keep_flag);
  CU(cudaGetLastError());
  *n_groups_out = n_groups;
  return CMX_OK;
}

static int pp_device(cmx_ctx *ctx, const PpParams &P, PpRecord *d_a, u64 *d_bca, u64 n, PpRecord *d_b, u64 *d_bcb, u64 *nsel_out,
                     const PpAbundance *wl = nullptr) {
  *nsel_out = 0;
  if (n == 0) return CMX_OK;
  if (n > 0x7FFFFFFFull) return fail(ctx, CMX_ERR_INVALID, "post-processing: more than 2^31-1 records in one call");
  const bool bc = P.kind == PP_BED_BC;
  cudaStream_t st = ctx->stream;
  DevMem<u64> d_k0, d_k1, d_nsel;
  DevMem<u32> d_i0, d_i1;
  DevMem<u8> d_head, d_keep;
  DevMem<> d_tmp;
  CU(d_k0.alloc(n * 8)); CU(d_k1.alloc(n * 8)); CU(d_i0.alloc(n * 4)); CU(d_i1.alloc(n * 4));
  CU(d_head.alloc(n)); CU(d_keep.alloc(n)); CU(d_nsel.alloc(16));
  const unsigned nb = (unsigned)((n + 255) / 256);
  if (!P.low_mem && P.tn5 && P.kind != PP_PAIRS) pp_tn5_kernel<<<nb, 256, 0, st>>>(P.kind, P.se, d_a, n);  // chromap.h:1322-1355: before the sort
  pp_iota_kernel<<<nb, 256, 0, st>>>(d_i0, n);
  cub::DoubleBuffer<u64> dk(d_k0, d_k1);
  cub::DoubleBuffer<u32> di(d_i0, d_i1);
  size_t tmp_bytes = 0, need = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, dk, di, (int)n, 0, 64, st);
  cub::DeviceSelect::Flagged(nullptr, need, d_a, d_keep.p, d_b, d_nsel.p, (int)n, st);
  tmp_bytes = std::max(tmp_bytes, need);
  cub::DeviceSelect::Flagged(nullptr, need, d_bca, d_keep.p, d_bcb, d_nsel.p, (int)n, st);
  tmp_bytes = std::max(tmp_bytes, need);
  if (P.bulk) tmp_bytes = std::max(tmp_bytes, pp_bulk_tmp_bytes(n, st));
  CU(d_tmp.alloc(tmp_bytes));
  // only the bits a key word can hold are sorted: word 0 (rid | start, or rid1 | rid2) up to its largest value in this call;
  // pp_key_word bounds the others: the 32-bit alignment lengths; length alone; mapq | direction | unique | read id
  u64 max0 = 0;
  CU(cudaMemsetAsync(d_nsel, 0, 16, st));
  pp_max_key0_kernel<<<std::min(nb, 1184u), 256, 0, st>>>(P.kind, d_a, n, d_nsel);
  CU(cudaMemcpyAsync(&max0, d_nsel, 8, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  int bits0 = 1;
  while (bits0 < 64 && (max0 >> bits0)) ++bits0;
  for (int w = pp_n_words(P.kind) - 1; w >= 0; --w) {  // least significant word first; every pass is stable
    pp_key_kernel<<<nb, 256, 0, st>>>(P.kind, w, d_a, bc ? d_bca : nullptr, di.Current(), n, dk.Current());
    int bits = 64;
    if (w == 0) bits = bits0;
    else if (P.kind == PP_PAIRS) bits = w == 2 ? 40 : 64;
    else if (bc) bits = w == 1 ? 16 : (w == 3 ? 56 : 64);
    else if (w == 2) bits = 32;
    CU(cub::DeviceRadixSort::SortPairs(d_tmp, tmp_bytes, dk, di, (int)n, 0, bits, st));
  }
  pp_gather_kernel<<<nb, 256, 0, st>>>(d_a, bc ? d_bca : nullptr, di.Current(), n, d_b, d_bcb);
  u64 n_res = n;  // entries of d_a / d_keep the compaction reads: one per record, or one per bulk group
  if (P.bulk) {
    const int rc = pp_bulk_resolve(ctx, P, *wl, d_b, d_bcb, n, d_k0, d_k1, d_i0, d_i1, d_tmp, d_a, d_bca, d_keep, &n_res);
    if (rc != CMX_OK) return rc;
  } else {
    pp_head_kernel<<<nb, 256, 0, st>>>(P.kind, P.se, P.dedup, d_b, bc ? d_bcb : nullptr, n, d_head);
    pp_resolve_kernel<<<nb, 256, 0, st>>>(P, d_b, bc ? d_bcb : nullptr, d_head, n, d_a, bc ? d_bca : nullptr, d_keep);
  }
  CU(cub::DeviceSelect::Flagged(d_tmp, tmp_bytes, d_a, d_keep.p, d_b, d_nsel.p, (int)n_res, st));
  if (bc) CU(cub::DeviceSelect::Flagged(d_tmp, tmp_bytes, d_bca, d_keep.p, d_bcb, d_nsel + 1, (int)n_res, st));
  u64 nsel = 0;
  CU(cudaMemcpyAsync(&nsel, d_nsel, 8, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  CU(cudaGetLastError());
  *nsel_out = nsel;
  return CMX_OK;
}

// The same in place on host buffers: same results as cmx_postprocess / cmx_postprocess_bc / cmx_postprocess_pairs
// (postprocess.cuh).  The record kind follows the context: pairs when output_format == 5, barcoded BED when
// barcode_keys != NULL, else bulk BED.
int cmx_postprocess_gpu(cmx_ctx *ctx, void *records, uint64_t *barcode_keys, uint64_t n, uint64_t *n_out) {
  if (!ctx || (!records && n) || !n_out) return CMX_ERR_INVALID;
  *n_out = 0;
  if (n == 0) return CMX_OK;
  if (n > 0x7FFFFFFFull) return fail(ctx, CMX_ERR_INVALID, "cmx_postprocess_gpu: more than 2^31-1 records in one call");
  CU(cudaSetDevice(ctx->device));
  const cmx_params &p = ctx->params;
  PpParams P;
  P.kind = p.output_format == 5 ? PP_PAIRS : (barcode_keys ? PP_BED_BC : (p.single_end ? PP_BED_SE : PP_BED));
  P.low_mem = p.low_memory_mode; P.dedup = p.remove_pcr_duplicates; P.tn5 = p.tn5_shift; P.mapq_threshold = p.mapq_threshold; P.se = p.single_end;
  if (P.kind == PP_PAIRS && barcode_keys) return fail(ctx, CMX_ERR_INVALID, "barcodes are not supported with pairs output");
  const bool bc = P.kind == PP_BED_BC;
  cudaStream_t st = ctx->stream;
  DevMem<PpRecord> d_a, d_b;
  DevMem<u64> d_bca, d_bcb;
  CU(d_a.alloc(n * sizeof(PpRecord))); CU(d_b.alloc(n * sizeof(PpRecord)));
  if (bc) { CU(d_bca.alloc(n * 8)); CU(d_bcb.alloc(n * 8)); }
  CU(cudaMemcpyAsync(d_a, records, n * sizeof(PpRecord), cudaMemcpyHostToDevice, st));
  if (bc) CU(cudaMemcpyAsync(d_bca, barcode_keys, n * 8, cudaMemcpyHostToDevice, st));
  u64 nsel = 0;
  const int rc = pp_device(ctx, P, d_a, d_bca, n, d_b, d_bcb, &nsel);
  if (rc != CMX_OK) return rc;
  if (nsel) CU(cudaMemcpyAsync(records, d_b, nsel * sizeof(PpRecord), cudaMemcpyDeviceToHost, st));
  if (bc && nsel) CU(cudaMemcpyAsync(barcode_keys, d_bcb, nsel * 8, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  *n_out = nsel;
  return CMX_OK;
}

// ---- --remove-pcr-duplicates-at-bulk-level for barcoded BED (mapping_writer.h:126-163, 166-376) ------------------------------
// Why a context cannot take the rule, or nullptr
static const char *bulk_dedup_refusal(const cmx_params &p) {
  if (!p.low_memory_mode) return "only the low-memory merge has bulk-level duplicate removal (in memory the reference removes duplicates per cell)";
  if (!p.remove_pcr_duplicates) return "the context does not remove duplicates";
  if (p.output_format == 4 || p.output_format == 5) return "bulk-level duplicate removal covers BED records, not SAM or pairs";
  return nullptr;
}
// The merge loop of ProcessAndOutputMappingsInLowMemory, one record at a time, over the records in the reference's order
static int postprocess_bc_bulk_host(const cmx_params &p, const std::unordered_map<uint64_t, uint32_t> &abundance, cmx_pe_record *recs, uint64_t *bcs,
                                    uint64_t n, uint64_t *n_out) {
  *n_out = 0;
  if (n == 0) return CMX_OK;
  std::vector<uint64_t> ord(n);
  for (uint64_t i = 0; i < n; ++i) ord[i] = i;
  auto key = [&](uint64_t i) {  // bed_mapping.h:32-37,145-153 prefixed by rid
    const cmx_pe_record &r = recs[i];
    return std::make_tuple(r.rid, r.fragment_start, r.fragment_length, bcs[i], r.mapq, r.direction, r.is_unique, r.read_id);
  };
  std::stable_sort(ord.begin(), ord.end(), [&](uint64_t a, uint64_t b) { return key(a) < key(b); });
  for (uint64_t i = 0; i < n; ++i)
    if (!abundance.count(bcs[i])) return CMX_ERR_INVALID;
  const bool se = p.single_end != 0;
  auto same_position = [&](uint64_t a, uint64_t b) {  // IsSamePosition, bed_mapping.h:43-45,155-158
    return recs[a].fragment_start == recs[b].fragment_start && (se || recs[a].fragment_length == recs[b].fragment_length);
  };
  auto same = [&](uint64_t a, uint64_t b) { return bcs[a] == bcs[b] && same_position(a, b); };  // operator==, bed_mapping.h:39-42,159-163
  struct Entry { uint64_t rec; uint32_t num_dups; };
  std::vector<Entry> entries;
  auto best = [&]() {  // FindBestMappingIndexFromDuplicates
    size_t b = 0;
    for (size_t k = 1; k < entries.size(); ++k) {
      const uint32_t ab = abundance.at(bcs[entries[k].rec]), bb = abundance.at(bcs[entries[b].rec]);
      if (entries[k].num_dups > entries[b].num_dups || (entries[k].num_dups == entries[b].num_dups && ab > bb)) b = k;
    }
    return entries[b].rec;
  };
  std::vector<cmx_pe_record> out_r;
  std::vector<uint64_t> out_b;
  auto emit = [&](uint64_t i, uint32_t dups) {
    cmx_pe_record r = recs[i];
    r.num_dups = (uint8_t)std::min<uint32_t>(255, dups);
    if (p.tn5_shift) { if (se) tn5_se(r); else tn5(r); }
    out_r.push_back(r); out_b.push_back(bcs[i]);
  };
  uint64_t last = 0;
  uint32_t num_last_dups = 0;
  for (uint64_t k = 0; k < n; ++k) {
    const uint64_t cur = ord[k];
    const bool duplicated = k > 0 && recs[cur].rid == recs[last].rid && (same(cur, last) || same_position(cur, last));
    if (duplicated) {
      ++num_last_dups;
      if (!entries.empty() && same(cur, entries.back().rec)) entries.back() = Entry{cur, 2};
      else entries.push_back(Entry{cur, 1});
      if (recs[cur].mapq > recs[last].mapq) last = cur;
    } else {
      if (k > 0) {
        last = best();
        entries.clear();
        if (recs[last].mapq >= p.mapq_threshold) emit(last, num_last_dups);
      }
      last = cur;
      num_last_dups = 1;
      entries.push_back(Entry{cur, 1});
    }
  }
  if (recs[last].mapq >= p.mapq_threshold) emit(best(), num_last_dups);  // the last group: tested before its best entry is chosen
  std::copy(out_r.begin(), out_r.end(), recs);
  std::copy(out_b.begin(), out_b.end(), bcs);
  *n_out = out_r.size();
  return CMX_OK;
}

int cmx_postprocess_bc_bulk(const cmx_params *p, const uint64_t *wl_keys, const uint32_t *wl_counts, uint64_t n_wl, cmx_pe_record *records,
                            uint64_t *barcode_keys, uint64_t n, uint64_t *n_out) {
  if (!p || (n_wl && (!wl_keys || !wl_counts)) || (n && (!records || !barcode_keys)) || !n_out) return CMX_ERR_INVALID;
  if (bulk_dedup_refusal(*p) || n > 0x7FFFFFFFull) return CMX_ERR_INVALID;
  if (n_wl == 0) return CMX_ERR_STATE;
  std::unordered_map<uint64_t, uint32_t> abundance;
  for (uint64_t i = 0; i < n_wl; ++i) abundance.emplace(wl_keys[i], wl_counts[i]);
  return postprocess_bc_bulk_host(*p, abundance, records, barcode_keys, n, n_out);
}

int cmx_postprocess_bc_bulk_gpu(cmx_ctx *ctx, cmx_pe_record *records, uint64_t *barcode_keys, uint64_t n, uint64_t *n_out) {
  if (!ctx || (n && (!records || !barcode_keys)) || !n_out) return CMX_ERR_INVALID;
  const cmx_params &p = ctx->params;
  if (const char *why = bulk_dedup_refusal(p)) return fail(ctx, CMX_ERR_INVALID, "cmx_postprocess_bc_bulk_gpu: %s", why);
  if (!ctx->wl_active) return fail(ctx, CMX_ERR_STATE, "cmx_postprocess_bc_bulk_gpu: no barcode whitelist uploaded; the rule ranks barcodes by their abundance in it");
  if (ctx->wl_output_nw)
    return fail(ctx, CMX_ERR_INVALID, "cmx_postprocess_bc_bulk_gpu: barcodes outside the whitelist (output_not_in_whitelist) have no abundance; the reference reads past its table for them");
  if (n > 0x7FFFFFFFull) return fail(ctx, CMX_ERR_INVALID, "cmx_postprocess_bc_bulk_gpu: more than 2^31-1 records in one call");
  *n_out = 0;
  if (n == 0) return CMX_OK;
  CU(cudaSetDevice(ctx->device));
  PpParams P;
  P.kind = PP_BED_BC; P.low_mem = 1; P.dedup = 1; P.tn5 = p.tn5_shift; P.mapq_threshold = p.mapq_threshold; P.se = p.single_end; P.bulk = 1;
  const PpAbundance wl{ctx->wl_slots, ctx->wl_n_slots - 1, table_shift(ctx->wl_n_slots), nullptr, ctx->wl_top_listed, ctx->wl_top_count};
  cudaStream_t st = ctx->stream;
  DevMem<PpRecord> d_a, d_b;
  DevMem<u64> d_bca, d_bcb;
  CU(d_a.alloc(n * sizeof(PpRecord))); CU(d_b.alloc(n * sizeof(PpRecord)));
  CU(d_bca.alloc(n * 8)); CU(d_bcb.alloc(n * 8));
  CU(cudaMemcpyAsync(d_a, records, n * sizeof(PpRecord), cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(d_bca, barcode_keys, n * 8, cudaMemcpyHostToDevice, st));
  u64 nsel = 0;
  const int rc = pp_device(ctx, P, d_a, d_bca, n, d_b, d_bcb, &nsel, &wl);
  if (rc != CMX_OK) return rc;
  if (nsel) CU(cudaMemcpyAsync(records, d_b, nsel * sizeof(PpRecord), cudaMemcpyDeviceToHost, st));
  if (nsel) CU(cudaMemcpyAsync(barcode_keys, d_bcb, nsel * 8, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  *n_out = nsel;
  return CMX_OK;
}

// ---- --allocate-multi-mappings (allocate.cuh) ------------------------------------------------------------------------------
// The checks both entries make before touching the records
static int allocation_refusal(cmx_ctx *ctx, const char *who, const cmx_pe_record *records, uint64_t n, int32_t distance, uint64_t *n_out) {
  if (!ctx || (!records && n) || !n_out) return CMX_ERR_INVALID;
  const cmx_params &p = ctx->params;
  if (p.low_memory_mode) return fail(ctx, CMX_ERR_INVALID, "%s: a low-memory context never allocates multi-mappings (the reference skips the step there)", who);
  if (p.output_format == 4 || p.output_format == 5)
    return fail(ctx, CMX_ERR_INVALID, "%s: multi-mapping allocation covers BED / TagAlign records, not SAM or pairs", who);
  if (distance < 0) return fail(ctx, CMX_ERR_INVALID, "%s: distance %d < 0 (the reference's uint32 cast would turn it into a wrap-around)", who, distance);
  if (n > 0x7FFFFFFFull) return fail(ctx, CMX_ERR_INVALID, "%s: more than 2^31-1 records in one call", who);
  return CMX_OK;
}
static const char *NO_MULTI = "%s: no multi-mapping (mapq < 4) among the records; the reference aborts here (mapping_processor.h:375)";

int cmx_allocate_multi_mappings(cmx_ctx *ctx, cmx_pe_record *records, uint64_t *barcode_keys, uint64_t n, int32_t distance, int32_t seed,
                                uint64_t *n_out, cmx_allocation_stats *stats) {
  const char *who = "cmx_allocate_multi_mappings";
  const int rc = allocation_refusal(ctx, who, records, n, distance, n_out);
  if (rc) return rc;
  const cmx_params &p = ctx->params;
  const bool bc = barcode_keys != nullptr;
  std::vector<cmx_pe_record> rr(records, records + n);
  std::vector<uint64_t> bb(bc ? barcode_keys : nullptr, bc ? barcode_keys + n : nullptr);
  cmx_params p1 = p;  // Tn5, sort, dedup; the MAPQ filter comes after the allocation
  p1.mapq_threshold = 0;
  uint64_t n1 = 0;
  if (bc) postprocess_bc_host(p1, rr.data(), bb.data(), n, &n1); else postprocess_host(p1, rr.data(), n, &n1);
  // uni records per sequence: starts (sorted: the records are) and ends in that order, ends sorted
  std::vector<uint8_t> keep(n1, 0);
  std::vector<uint64_t> us, ue_s;
  std::vector<uint32_t> multi;
  for (uint64_t i = 0; i < n1; ++i) {
    const uint64_t rid = (uint64_t)rr[i].rid << 32;
    if (rr[i].mapq < 4) { multi.push_back((uint32_t)i); continue; }
    keep[i] = 1;
    us.push_back(rid | rr[i].fragment_start);
    ue_s.push_back(rid | (uint32_t)(rr[i].fragment_start + rr[i].fragment_length));
  }
  if (multi.empty()) return fail(ctx, CMX_ERR_INVALID, NO_MULTI, who);
  std::vector<uint64_t> ue = ue_s;
  std::sort(ue.begin(), ue.end());
  std::stable_sort(multi.begin(), multi.end(), [&](uint32_t a, uint32_t b) { return rr[a].read_id < rr[b].read_id; });
  auto weight = [&](const cmx_pe_record &r) -> uint32_t {  // mapping_processor.h:255-317
    const uint64_t rid = (uint64_t)r.rid << 32;
    const uint32_t d = (uint32_t)distance, start = r.fragment_start, end = start + r.fragment_length;
    const uint32_t qs = start > d ? start - d : 0u, qe = end + d;
    const uint64_t lo = std::lower_bound(us.begin(), us.end(), rid) - us.begin(), a = std::lower_bound(us.begin(), us.end(), rid | qe) - us.begin();
    if (qe > qs)
      return (uint32_t)((a - lo) - (uint64_t)(std::lower_bound(ue.begin(), ue.end(), rid | (qs + 1u)) - std::lower_bound(ue.begin(), ue.end(), rid)));
    uint32_t c = 0;  // end + d wrapped: only uni records starting within AL_MAX_LEN of qs can end past it
    const uint64_t i0 = std::max<uint64_t>(lo, std::lower_bound(us.begin(), us.end(), rid | (qs > AL_MAX_LEN ? qs - AL_MAX_LEN : 0u)) - us.begin());
    for (uint64_t i = i0; i < a; ++i) c += (uint32_t)ue_s[i] > qs;
    return c;
  };
  std::mt19937 generator(seed);
  cmx_allocation_stats st{};
  st.n_multi = multi.size();
  std::vector<uint32_t> weights;
  for (size_t s = 0; s < multi.size();) {  // one read: candidates multi[s, e)
    size_t e = s;
    uint32_t sum = 0;
    weights.clear();
    for (; e < multi.size() && rr[multi[e]].read_id == rr[multi[s]].read_id; ++e) { weights.push_back(weight(rr[multi[e]])); sum += weights.back(); }
    if (sum == 0) ++st.n_without_overlap;
    else {
      std::discrete_distribution<uint32_t> distribution(weights.begin(), weights.end());
      keep[multi[s + distribution(generator)]] = 1;
      ++st.n_allocated;
      st.n_draws += weights.size() >= 2;
    }
    s = e;
  }
  uint64_t n2 = 0;
  for (uint64_t i = 0; i < n1; ++i)
    if (keep[i]) { rr[n2] = rr[i]; if (bc) bb[n2] = bb[i]; ++n2; }
  for (uint64_t i = 0; i < n2; ++i) { if (rr[i].is_unique == 1) ++st.n_uni_after; else ++st.n_multi_after; }
  cmx_params p2 = p;  // sort again, MAPQ filter
  p2.remove_pcr_duplicates = 0; p2.tn5_shift = 0;
  uint64_t n3 = 0;
  if (bc) postprocess_bc_host(p2, rr.data(), bb.data(), n2, &n3); else postprocess_host(p2, rr.data(), n2, &n3);
  std::copy(rr.begin(), rr.begin() + n3, records);
  if (bc) std::copy(bb.begin(), bb.begin() + n3, barcode_keys);
  *n_out = n3;
  if (stats) *stats = st;
  return CMX_OK;
}

int cmx_allocate_multi_mappings_gpu(cmx_ctx *ctx, cmx_pe_record *records, uint64_t *barcode_keys, uint64_t n, int32_t distance, int32_t seed,
                                    uint64_t *n_out, cmx_allocation_stats *stats) {
  const char *who = "cmx_allocate_multi_mappings_gpu";
  const int rc0 = allocation_refusal(ctx, who, records, n, distance, n_out);
  if (rc0) return rc0;
  if (n == 0) return fail(ctx, CMX_ERR_INVALID, NO_MULTI, who);
  CU(cudaSetDevice(ctx->device));
  const cmx_params &p = ctx->params;
  const bool bc = barcode_keys != nullptr;
  PpParams P;
  P.kind = bc ? PP_BED_BC : (p.single_end ? PP_BED_SE : PP_BED);
  P.low_mem = 0; P.dedup = p.remove_pcr_duplicates; P.tn5 = p.tn5_shift; P.mapq_threshold = 0; P.se = p.single_end;
  cudaStream_t st = ctx->stream;
  DevMem<PpRecord> d_a, d_b;
  DevMem<u64> d_bca, d_bcb;
  CU(d_a.alloc(n * sizeof(PpRecord))); CU(d_b.alloc(n * sizeof(PpRecord)));
  if (bc) { CU(d_bca.alloc(n * 8)); CU(d_bcb.alloc(n * 8)); }
  CU(cudaMemcpyAsync(d_a, records, n * sizeof(PpRecord), cudaMemcpyHostToDevice, st));
  if (bc) CU(cudaMemcpyAsync(d_bca, barcode_keys, n * 8, cudaMemcpyHostToDevice, st));
  u64 n1 = 0;
  int rc = pp_device(ctx, P, d_a, d_bca, n, d_b, d_bcb, &n1);  // sorted, deduplicated: d_b[0, n1)
  if (rc != CMX_OK) return rc;
  // 1. split
  DevMem<u8> d_uni, d_multi;
  DevMem<u64> d_ks, d_ke, d_us, d_ue_s, d_ue, d_cnt;
  DevMem<u32> d_midx;
  DevMem<> d_tmp;
  CU(d_uni.alloc(n1 + 1)); CU(d_multi.alloc(n1 + 1)); CU(d_ks.alloc(n1 * 8)); CU(d_ke.alloc(n1 * 8));
  CU(d_us.alloc(n1 * 8)); CU(d_ue_s.alloc(n1 * 8)); CU(d_ue.alloc(n1 * 8)); CU(d_midx.alloc(n1 * 4)); CU(d_cnt.alloc(32));
  const unsigned nb1 = (unsigned)((n1 + 255) / 256);
  al_split_kernel<<<nb1, 256, 0, st>>>(d_b, n1, d_uni, d_multi, d_ks, d_ke);
  thrust::counting_iterator<u32> iota(0u);
  size_t tmp_bytes = 0, need = 0;
  CU(cub::DeviceSelect::Flagged(nullptr, need, d_ks.p, d_uni.p, d_us.p, d_cnt.p, (int)n1, st)); tmp_bytes = std::max(tmp_bytes, need);
  CU(cub::DeviceSelect::Flagged(nullptr, need, iota, d_multi.p, d_midx.p, d_cnt.p, (int)n1, st)); tmp_bytes = std::max(tmp_bytes, need);
  CU(cub::DeviceRadixSort::SortKeys(nullptr, need, d_ue_s.p, d_ue.p, (int)n1, 0, 64, st)); tmp_bytes = std::max(tmp_bytes, need);
  CU(cub::DeviceRadixSort::SortPairs(nullptr, need, (u32 *)nullptr, (u32 *)nullptr, (u32 *)nullptr, (u32 *)nullptr, (int)n1, 0, 32, st)); tmp_bytes = std::max(tmp_bytes, need);
  CU(cub::DeviceScan::ExclusiveSum(nullptr, need, (u32 *)nullptr, (u32 *)nullptr, (int)n1, st)); tmp_bytes = std::max(tmp_bytes, need);
  CU(cub::DeviceSelect::Flagged(nullptr, need, d_b.p, d_uni.p, d_a.p, d_cnt.p, (int)n1, st)); tmp_bytes = std::max(tmp_bytes, need);
  CU(cub::DeviceSelect::Flagged(nullptr, need, d_bcb.p, d_uni.p, d_bca.p, d_cnt.p, (int)n1, st)); tmp_bytes = std::max(tmp_bytes, need);
  CU(d_tmp.alloc(tmp_bytes));
  CU(cudaMemsetAsync(d_cnt, 0, 32, st));
  CU(cub::DeviceSelect::Flagged(d_tmp, tmp_bytes, d_ks.p, d_uni.p, d_us.p, d_cnt.p, (int)n1, st));
  CU(cub::DeviceSelect::Flagged(d_tmp, tmp_bytes, d_ke.p, d_uni.p, d_ue_s.p, d_cnt.p, (int)n1, st));
  CU(cub::DeviceSelect::Flagged(d_tmp, tmp_bytes, iota, d_multi.p, d_midx.p, d_cnt + 1, (int)n1, st));
  u64 cnt[2] = {0, 0};
  CU(cudaMemcpyAsync(cnt, d_cnt, 16, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  const u32 n_uni = (u32)cnt[0], m = (u32)cnt[1];
  if (m == 0) return fail(ctx, CMX_ERR_INVALID, NO_MULTI, who);
  // 2. weights
  if (n_uni) CU(cub::DeviceRadixSort::SortKeys(d_tmp, tmp_bytes, d_ue_s.p, d_ue.p, (int)n_uni, 0, 64, st));
  DevMem<u32> d_w, d_rk, d_rk2, d_j, d_perm, d_ws, d_rs, d_draws, d_didx, d_stream;
  DevMem<u8> d_head, d_kept;
  CU(d_w.alloc(m * 4ull)); CU(d_rk.alloc(m * 4ull)); CU(d_rk2.alloc(m * 4ull)); CU(d_j.alloc(m * 4ull)); CU(d_perm.alloc(m * 4ull));
  CU(d_ws.alloc(m * 4ull)); CU(d_rs.alloc(m * 4ull)); CU(d_draws.alloc(m * 4ull)); CU(d_didx.alloc(m * 4ull)); CU(d_head.alloc(m)); CU(d_kept.alloc(m));
  const unsigned nbm = (m + 255) / 256;
  al_count_kernel<<<nbm, 256, 0, st>>>(d_b, d_midx, m, d_us, d_ue_s, d_ue, n_uni, (u32)distance, d_w, d_rk);
  CU(cudaGetLastError());
  // 3. group by read (stable), heads, per read counts, draw indices
  pp_iota_kernel<<<nbm, 256, 0, st>>>(d_j, m);
  CU(cub::DeviceRadixSort::SortPairs(d_tmp, tmp_bytes, d_rk.p, d_rk2.p, d_j.p, d_perm.p, (int)m, 0, 32, st));
  al_head_kernel<<<nbm, 256, 0, st>>>(d_rk2, d_perm, d_w, m, d_head, d_ws);
  CU(cub::DeviceSelect::Flagged(d_tmp, tmp_bytes, iota, d_head.p, d_rs.p, d_cnt + 2, (int)m, st));
  CU(cudaMemcpyAsync(cnt, d_cnt + 2, 8, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  const u32 n_reads = (u32)cnt[0];
  const unsigned nbr = (n_reads + 255) / 256;
  al_read_kernel<<<nbr, 256, 0, st>>>(d_rs, n_reads, m, d_ws, d_draws, d_kept);
  CU(cudaGetLastError());
  CU(cub::DeviceScan::ExclusiveSum(d_tmp, tmp_bytes, d_draws.p, d_didx.p, (int)n_reads, st));
  u32 last[2] = {0, 0};
  CU(cudaMemcpyAsync(&last[0], d_didx + (n_reads - 1), 4, cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(&last[1], d_draws + (n_reads - 1), 4, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  const u64 n_draws = (u64)last[0] + last[1];
  // 4. the generator stream
  if (n_draws) {
    std::vector<u32> mt(624);
    mt_seed_fill(mt.data(), (u32)seed);
    DevMem<u32> d_mt;
    CU(d_mt.alloc(624 * 4)); CU(d_stream.alloc(2 * n_draws * 4));
    CU(cudaMemcpyAsync(d_mt, mt.data(), 624 * 4, cudaMemcpyHostToDevice, st));
    al_mt_kernel<<<1, 256, 0, st>>>(d_mt, 2 * n_draws, d_stream);
    CU(cudaStreamSynchronize(st));  // d_mt's host copy lives in this block
  }
  // 5. the draws: keep = uni flags + picked candidates
  al_draw_kernel<<<nbr, 256, 0, st>>>(d_rs, n_reads, m, d_ws, d_perm, d_midx, d_draws, d_didx, d_kept, d_stream, d_uni);
  CU(cudaGetLastError());
  // 6. compact into d_a, count is_unique, sort again and filter
  CU(cub::DeviceSelect::Flagged(d_tmp, tmp_bytes, d_b.p, d_uni.p, d_a.p, d_cnt + 3, (int)n1, st));
  if (bc) CU(cub::DeviceSelect::Flagged(d_tmp, tmp_bytes, d_bcb.p, d_uni.p, d_bca.p, d_cnt + 3, (int)n1, st));
  CU(cudaMemcpyAsync(cnt, d_cnt + 3, 8, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  const u64 n2 = cnt[0];
  CU(cudaMemsetAsync(d_cnt + 3, 0, 8, st));
  if (n2) al_unique_count_kernel<<<(unsigned)((n2 + 255) / 256), 256, 0, st>>>(d_a, n2, (unsigned long long *)(d_cnt.p + 3));  // n2 == 0: no uni record, no read kept
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(cnt + 1, d_cnt + 3, 8, cudaMemcpyDeviceToHost, st));
  P.dedup = 0; P.tn5 = 0; P.mapq_threshold = p.mapq_threshold;
  u64 n3 = 0;
  rc = pp_device(ctx, P, d_a, d_bca, n2, d_b, d_bcb, &n3);  // waits for the stream
  if (rc != CMX_OK) return rc;
  if (n3) CU(cudaMemcpyAsync(records, d_b, n3 * sizeof(PpRecord), cudaMemcpyDeviceToHost, st));
  if (bc && n3) CU(cudaMemcpyAsync(barcode_keys, d_bcb, n3 * 8, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  CU(cudaGetLastError());
  *n_out = n3;
  if (stats) {
    stats->n_multi = m; stats->n_allocated = n2 - n_uni; stats->n_without_overlap = n_reads - (n2 - n_uni); stats->n_draws = n_draws;
    stats->n_uni_after = cnt[1]; stats->n_multi_after = n2 - cnt[1];
  }
  return CMX_OK;
}

// ---- multi-GPU duplicate-removal exchange (SURVEY.md §8e, exchange.cuh) -------------------------------------------------
// NCCL is reached through dlopen: the library has no link-time dependency on it, and inside a process that already
// holds an NCCL (PyTorch's) that copy is the one used.  Types are declared here (ABI of nccl.h 2.x).
namespace {
struct NcclApi {
  typedef struct { char internal[128]; } UniqueId;
  int (*GetUniqueId)(UniqueId *) = nullptr;
  int (*CommInitRank)(void **, int, UniqueId, int) = nullptr;
  int (*CommDestroy)(void *) = nullptr;
  int (*AllGather)(const void *, void *, size_t, int, void *, cudaStream_t) = nullptr;
  int (*Send)(const void *, size_t, int, int, void *, cudaStream_t) = nullptr;
  int (*Recv)(void *, size_t, int, int, void *, cudaStream_t) = nullptr;
  int (*GroupStart)() = nullptr;
  int (*GroupEnd)() = nullptr;
  const char *(*GetErrorString)(int) = nullptr;
  bool ok = false;
  std::string why;
};
NcclApi &nccl_api() {
  static NcclApi api;
  static bool tried = false;
  if (tried) return api;
  tried = true;
  // an NCCL the process already holds (PyTorch's) first; otherwise CMX_NCCL_LIB, then the system library.  RTLD_LOCAL: our copy
  // must not satisfy the symbol lookups of a framework that is loaded later and expects its own (newer) NCCL.
  void *h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD | RTLD_LOCAL);
  if (!h) { const char *pth = getenv("CMX_NCCL_LIB"); if (pth && *pth) h = dlopen(pth, RTLD_NOW | RTLD_LOCAL); }
  if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_LOCAL);
  if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_LOCAL);
  if (!h) { api.why = std::string("libnccl.so.2 not found: ") + dlerror(); return api; }
  api.GetUniqueId = (int (*)(NcclApi::UniqueId *))dlsym(h, "ncclGetUniqueId");
  api.CommInitRank = (int (*)(void **, int, NcclApi::UniqueId, int))dlsym(h, "ncclCommInitRank");
  api.CommDestroy = (int (*)(void *))dlsym(h, "ncclCommDestroy");
  api.AllGather = (int (*)(const void *, void *, size_t, int, void *, cudaStream_t))dlsym(h, "ncclAllGather");
  api.Send = (int (*)(const void *, size_t, int, int, void *, cudaStream_t))dlsym(h, "ncclSend");
  api.Recv = (int (*)(void *, size_t, int, int, void *, cudaStream_t))dlsym(h, "ncclRecv");
  api.GroupStart = (int (*)())dlsym(h, "ncclGroupStart");
  api.GroupEnd = (int (*)())dlsym(h, "ncclGroupEnd");
  api.GetErrorString = (const char *(*)(int))dlsym(h, "ncclGetErrorString");
  api.ok = api.GetUniqueId && api.CommInitRank && api.CommDestroy && api.AllGather && api.Send && api.Recv && api.GroupStart && api.GroupEnd;
  if (!api.ok) api.why = "libnccl.so.2 lacks the expected symbols";
  return api;
}
const int NCCL_UINT8 = 1, NCCL_UINT64 = 5;  // ncclDataType_t
}  // namespace

#define NC(call)                                                                                                      \
  do {                                                                                                                \
    const int r_ = (call);                                                                                            \
    if (r_ != 0)                                                                                                      \
      return fail(ctx, CMX_ERR_CUDA, "%s:%d %s: %s", __FILE__, __LINE__, #call,                                       \
                  nccl_api().GetErrorString ? nccl_api().GetErrorString(r_) : "NCCL error");                          \
  } while (0)

int cmx_comm_unique_id(void *id128) {
  if (!id128) return CMX_ERR_INVALID;
  NcclApi &N = nccl_api();
  if (!N.ok) return CMX_ERR_STATE;
  NcclApi::UniqueId id;
  if (N.GetUniqueId(&id) != 0) return CMX_ERR_CUDA;
  memcpy(id128, &id, 128);
  return CMX_OK;
}

int cmx_comm_init(cmx_ctx *ctx, int n_ranks, int rank, const void *id128) {
  if (!ctx || !id128 || n_ranks < 1 || rank < 0 || rank >= n_ranks) return CMX_ERR_INVALID;
  NcclApi &N = nccl_api();
  if (!N.ok) return fail(ctx, CMX_ERR_STATE, "NCCL unavailable: %s", N.why.c_str());
  CU(cudaSetDevice(ctx->device));
  if (ctx->nccl_comm) { N.CommDestroy(ctx->nccl_comm); ctx->nccl_comm = nullptr; }
  NcclApi::UniqueId id;
  memcpy(&id, id128, 128);
  const int rc = N.CommInitRank(&ctx->nccl_comm, n_ranks, id, rank);
  if (rc != 0) return fail(ctx, CMX_ERR_CUDA, "ncclCommInitRank: %s", N.GetErrorString ? N.GetErrorString(rc) : "error");
  ctx->comm_rank = rank; ctx->comm_size = n_ranks;
  return CMX_OK;
}

int cmx_comm_destroy(cmx_ctx *ctx) {
  if (!ctx) return CMX_ERR_INVALID;
  if (ctx->nccl_comm) { nccl_api().CommDestroy(ctx->nccl_comm); ctx->nccl_comm = nullptr; }
  ctx->comm_rank = 0; ctx->comm_size = 1;
  return CMX_OK;
}

// This rank's records in, this rank's survivors out (reference order, duplicate counts set, MAPQ-filtered, Tn5 NOT yet
// applied: the low-memory merge shifts after the final ordering, mapping_writer.h:285-287 — cmx_exchange_finish below).
int cmx_dedup_exchange(cmx_ctx *ctx, const void *records, const uint64_t *barcode_keys, uint64_t n, int on_device, void *out_records,
                       uint64_t *out_barcode_keys, uint64_t *n_out, cmx_exchange_stats *stats) {
  if (!ctx || (!records && n) || !out_records || !n_out) return CMX_ERR_INVALID;
  *n_out = 0;
  if (stats) memset(stats, 0, sizeof(*stats));
  const cmx_params &p = ctx->params;
  if (p.output_format == 5 || p.single_end || !p.low_memory_mode)
    return fail(ctx, CMX_ERR_INVALID, "cmx_dedup_exchange: paired-end BED records in low-memory mode only (every preset with duplicate removal)");
  if (!ctx->nccl_comm) return fail(ctx, CMX_ERR_STATE, "cmx_dedup_exchange: cmx_comm_init first");
  if (n >= 0x7FFFFFFFull) return fail(ctx, CMX_ERR_INVALID, "cmx_dedup_exchange: more than 2^31-1 records on one rank");
  NcclApi &N = nccl_api();
  CU(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const bool bc = barcode_keys != nullptr;
  const int tw = bc ? 3 : 2, R = ctx->comm_size, rank = ctx->comm_rank;
  PpRecord *d_rec = nullptr, *d_out = nullptr;  // the caller's device buffers, or copies of its host records
  u64 *d_bc = nullptr, *d_outbc = nullptr;
  DevMem<PpRecord> rec_copy, out_copy;
  DevMem<u64> bc_copy, outbc_copy, d_cnt, d_send, d_all, d_k0, d_k1, d_nsel;
  DevMem<u32> d_i0, d_i1, d_sel, d_selc;
  DevMem<u8> d_head, d_keep, d_dups, d_dupsc;
  DevMem<> d_tmp;
  Event ev[4];
  for (auto &e : ev) CU(e.alloc(cudaEventDefault));
  if (on_device) { d_rec = (PpRecord *)records; d_bc = (u64 *)barcode_keys; d_out = (PpRecord *)out_records; d_outbc = (u64 *)out_barcode_keys; }
  else {
    CU(rec_copy.alloc(std::max<u64>(n, 1) * sizeof(PpRecord))); CU(out_copy.alloc(std::max<u64>(n, 1) * sizeof(PpRecord)));
    d_rec = rec_copy; d_out = out_copy;
    CU(cudaMemcpyAsync(d_rec, records, n * sizeof(PpRecord), cudaMemcpyHostToDevice, st));
    if (bc) {
      CU(bc_copy.alloc(std::max<u64>(n, 1) * 8)); CU(outbc_copy.alloc(std::max<u64>(n, 1) * 8));
      d_bc = bc_copy; d_outbc = outbc_copy;
      CU(cudaMemcpyAsync(d_bc, barcode_keys, n * 8, cudaMemcpyHostToDevice, st));
    }
  }
  // sizes: an 8-byte all-gather of the record counts
  CU(d_cnt.alloc((size_t)(R + 1) * 8));
  CU(cudaMemcpyAsync(d_cnt + R, &n, 8, cudaMemcpyHostToDevice, st));
  NC(N.AllGather(d_cnt + R, d_cnt, 1, NCCL_UINT64, ctx->nccl_comm, st));
  std::vector<u64> cnt(R);
  CU(cudaMemcpyAsync(cnt.data(), d_cnt, (size_t)R * 8, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  u64 n_pad = 1, n_total = 0;
  for (u64 c : cnt) { n_pad = std::max(n_pad, c); n_total += c; }
  const u64 n_all = n_pad * (u64)R;
  if (n_all >= 0xFFFFFFFFull) return fail(ctx, CMX_ERR_INVALID, "cmx_dedup_exchange: %llu gathered tuples exceed 2^32", (unsigned long long)n_all);
  // pack -> ONE all-gather of the tuples -> sort -> decide
  CU(d_send.alloc(n_pad * tw * 8)); CU(d_all.alloc(n_all * tw * 8));
  CU(d_k0.alloc(n_all * 8)); CU(d_k1.alloc(n_all * 8)); CU(d_i0.alloc(n_all * 4)); CU(d_i1.alloc(n_all * 4));
  CU(d_head.alloc(n_all)); CU(d_keep.alloc(n_all)); CU(d_dups.alloc(n_all)); CU(d_dupsc.alloc(std::max<u64>(n, 1)));
  CU(d_sel.alloc(n_all * 4)); CU(d_selc.alloc(std::max<u64>(n, 1) * 4)); CU(d_nsel.alloc(16));
  CU(cudaEventRecord(ev[0], st));
  ex_pack_kernel<<<(unsigned)((n_pad + 255) / 256), 256, 0, st>>>(d_rec, d_bc, n, n_pad, bc ? 1 : 0, d_send);
  CU(cudaEventRecord(ev[1], st));
  NC(N.AllGather(d_send, d_all, n_pad * tw * 8, NCCL_UINT8, ctx->nccl_comm, st));
  CU(cudaEventRecord(ev[2], st));
  const unsigned nb = (unsigned)((n_all + 255) / 256);
  pp_iota_kernel<<<nb, 256, 0, st>>>(d_i0, n_all);
  cub::DoubleBuffer<u64> dk(d_k0, d_k1);
  cub::DoubleBuffer<u32> di(d_i0, d_i1);
  size_t tmp_bytes = 0, need = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, dk, di, (int)n_all, 0, 64, st);
  cub::DeviceSelect::Flagged(nullptr, need, d_sel.p, d_keep.p, d_selc.p, d_nsel.p, (int)n_all, st);
  tmp_bytes = std::max(tmp_bytes, need);
  CU(d_tmp.alloc(tmp_bytes));
  // least significant key first, every pass stable: bulk (b, a); barcoded (low 48 bits of b, barcode, length, a)
  const int passes_bulk[2] = {4, 3}, passes_bc[4] = {0, 1, 2, 3};
  for (int q = 0; q < (bc ? 4 : 2); ++q) {
    const int pass = bc ? passes_bc[q] : passes_bulk[q];
    ex_key_kernel<<<nb, 256, 0, st>>>(d_all, tw, pass, di.Current(), n_all, dk.Current());
    CU(cub::DeviceRadixSort::SortPairs(d_tmp, tmp_bytes, dk, di, (int)n_all, 0, pass == 2 ? 16 : 64, st));
  }
  // padding sorts last (a = ~0): only the first n_total sorted entries are records
  if (n_total) {
    const unsigned nbt = (unsigned)((n_total + 255) / 256);
    ex_head_kernel<<<nbt, 256, 0, st>>>(d_all, tw, p.remove_pcr_duplicates, di.Current(), n_total, d_head);
    ex_resolve_kernel<<<nbt, 256, 0, st>>>(d_all, tw, di.Current(), d_head, n_total, n_pad, rank, p.mapq_threshold, d_keep, d_sel, d_dups);
    CU(cub::DeviceSelect::Flagged(d_tmp, tmp_bytes, d_sel.p, d_keep.p, d_selc.p, d_nsel.p, (int)n_total, st));
    CU(cub::DeviceSelect::Flagged(d_tmp, tmp_bytes, d_dups.p, d_keep.p, d_dupsc.p, d_nsel + 1, (int)n_total, st));
  } else CU(cudaMemsetAsync(d_nsel, 0, 16, st));
  u64 nsel = 0;
  CU(cudaMemcpyAsync(&nsel, d_nsel, 8, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  if (nsel) ex_gather_kernel<<<(unsigned)((nsel + 255) / 256), 256, 0, st>>>(d_rec, d_bc, d_selc, d_dupsc, p.remove_pcr_duplicates, nsel, d_out, bc ? d_outbc : nullptr);
  CU(cudaEventRecord(ev[3], st));
  if (!on_device && nsel) {
    CU(cudaMemcpyAsync(out_records, d_out, nsel * sizeof(PpRecord), cudaMemcpyDeviceToHost, st));
    if (bc && out_barcode_keys) CU(cudaMemcpyAsync(out_barcode_keys, d_outbc, nsel * 8, cudaMemcpyDeviceToHost, st));
  }
  CU(cudaStreamSynchronize(st));
  CU(cudaGetLastError());
  if (stats) {
    cudaEventElapsedTime(&stats->pack_ms, ev[0], ev[1]);
    cudaEventElapsedTime(&stats->allgather_ms, ev[1], ev[2]);
    cudaEventElapsedTime(&stats->resolve_ms, ev[2], ev[3]);
    stats->bytes_sent = n_pad * tw * 8; stats->bytes_received = n_all * tw * 8; stats->n_global = n_total; stats->n_ranks = (uint32_t)R;
  }
  *n_out = nsel;
  return CMX_OK;
}

// The same step as a range shuffle (exchange.cuh, second half): this rank's records in; out = the records of THIS RANK'S KEY
// RANGE after duplicate removal over the whole run, in the reference's order, num_dups set, MAPQ-filtered, Tn5 applied —
// the run's output is the ranks' outputs one after the other in rank order.  Work per rank is proportional to its share of
// the run (the all-gather variant above sorts every rank's tuples on every rank).
int cmx_dedup_shuffle(cmx_ctx *ctx, const void *records, const uint64_t *barcode_keys, uint64_t n, int on_device, void *out_records,
                      uint64_t *out_barcode_keys, uint64_t out_capacity, uint64_t *n_out, cmx_shuffle_stats *stats) {
  if (!ctx || (!records && n) || (!out_records && out_capacity) || !n_out) return CMX_ERR_INVALID;
  *n_out = 0;
  if (stats) memset(stats, 0, sizeof(*stats));
  const cmx_params &p = ctx->params;
  if (p.output_format == 5 || p.single_end || !p.low_memory_mode)
    return fail(ctx, CMX_ERR_INVALID, "cmx_dedup_shuffle: paired-end BED records in low-memory mode only (every preset with duplicate removal)");
  if (!ctx->nccl_comm) return fail(ctx, CMX_ERR_STATE, "cmx_dedup_shuffle: cmx_comm_init first");
  if (n >= 0x7FFFFFFFull) return fail(ctx, CMX_ERR_INVALID, "cmx_dedup_shuffle: more than 2^31-1 records on one rank");
  NcclApi &N = nccl_api();
  CU(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const bool bc = barcode_keys != nullptr;
  const int R = ctx->comm_size, rank = ctx->comm_rank;
  PpRecord *d_rec = nullptr;  // the caller's device records, or a copy of its host records
  u64 *d_bc = nullptr;
  DevMem<PpRecord> rec_copy, d_send, d_recv, d_res;
  DevMem<u64> bc_copy, d_sendbc, d_recvbc, d_resbc, d_a, d_samp, d_all0, d_all1, d_split, d_off, d_offall;
  DevMem<u32> d_d0, d_d1, d_i0, d_i1;
  DevMem<> d_tmp;
  Event ev[4];
  for (auto &e : ev) CU(e.alloc(cudaEventDefault));
  const u64 n1 = std::max<u64>(n, 1);
  if (on_device) { d_rec = (PpRecord *)records; d_bc = (u64 *)barcode_keys; }
  else {
    CU(rec_copy.alloc(n1 * sizeof(PpRecord)));
    d_rec = rec_copy;
    CU(cudaMemcpyAsync(d_rec, records, n * sizeof(PpRecord), cudaMemcpyHostToDevice, st));
    if (bc) { CU(bc_copy.alloc(n1 * 8)); d_bc = bc_copy; CU(cudaMemcpyAsync(d_bc, barcode_keys, n * 8, cudaMemcpyHostToDevice, st)); }
  }
  const u64 n_samp = (u64)R * SH_SAMPLE;
  CU(d_a.alloc(n1 * 8)); CU(d_samp.alloc(SH_SAMPLE * 8)); CU(d_all0.alloc(n_samp * 8)); CU(d_all1.alloc(n_samp * 8));
  CU(d_split.alloc((size_t)std::max(R - 1, 1) * 8)); CU(d_off.alloc((size_t)(R + 1) * 8)); CU(d_offall.alloc((size_t)R * (R + 1) * 8));
  CU(d_d0.alloc(n1 * 4)); CU(d_d1.alloc(n1 * 4)); CU(d_i0.alloc(n1 * 4)); CU(d_i1.alloc(n1 * 4));
  CU(d_send.alloc(n1 * sizeof(PpRecord)));
  if (bc) CU(d_sendbc.alloc(n1 * 8));
  size_t tmp_bytes = 0, need = 0;
  {
    cub::DoubleBuffer<u64> ks(d_all0, d_all1);
    cub::DeviceRadixSort::SortKeys(nullptr, tmp_bytes, ks, (int)n_samp, 0, 64, st);
    cub::DoubleBuffer<u32> dd(d_d0, d_d1), di(d_i0, d_i1);
    cub::DeviceRadixSort::SortPairs(nullptr, need, dd, di, (int)n1, 0, 32, st);
    tmp_bytes = std::max(tmp_bytes, need);
  }
  CU(d_tmp.alloc(tmp_bytes));
  // ---- partition: splitters from an all-gathered sample, destination of every record, records grouped by destination
  CU(cudaEventRecord(ev[0], st));
  const unsigned nb = (unsigned)((n1 + 255) / 256);
  if (n) sh_key_kernel<<<nb, 256, 0, st>>>(d_rec, n, d_a);
  sh_sample_kernel<<<(SH_SAMPLE + 255) / 256, 256, 0, st>>>(d_a, n, d_samp);
  NC(N.AllGather(d_samp, d_all0, SH_SAMPLE, NCCL_UINT64, ctx->nccl_comm, st));
  cub::DoubleBuffer<u64> ks(d_all0, d_all1);
  CU(cub::DeviceRadixSort::SortKeys(d_tmp, tmp_bytes, ks, (int)n_samp, 0, 64, st));
  std::vector<u64> samp(n_samp), split(std::max(R - 1, 1), 0);
  CU(cudaMemcpyAsync(samp.data(), ks.Current(), n_samp * 8, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  const u64 valid = (u64)(std::lower_bound(samp.begin(), samp.end(), (u64)EX_PAD) - samp.begin());  // padding sorts last
  for (int j = 1; j < R; ++j) split[j - 1] = valid ? samp[valid * (u64)j / (u64)R] : 0ull;           // the same on every rank
  CU(cudaMemcpyAsync(d_split, split.data(), split.size() * 8, cudaMemcpyHostToDevice, st));
  int dest_bits = 1;
  while ((1 << dest_bits) < R) ++dest_bits;
  cub::DoubleBuffer<u32> dd(d_d0, d_d1), di(d_i0, d_i1);
  if (n) {
    sh_dest_kernel<<<nb, 256, 0, st>>>(d_a, n, d_split, R - 1, dd.Current());
    pp_iota_kernel<<<nb, 256, 0, st>>>(di.Current(), n);
    CU(cub::DeviceRadixSort::SortPairs(d_tmp, tmp_bytes, dd, di, (int)n, 0, dest_bits, st));  // stable: mapping order kept inside a destination
    pp_gather_kernel<<<nb, 256, 0, st>>>(d_rec, bc ? d_bc : nullptr, di.Current(), n, d_send, d_sendbc);
  }
  sh_bounds_kernel<<<(R + 1 + 63) / 64, 64, 0, st>>>(dd.Current(), n, R, d_off);
  NC(N.AllGather(d_off, d_offall, (size_t)(R + 1), NCCL_UINT64, ctx->nccl_comm, st));
  std::vector<u64> offall((size_t)R * (R + 1));
  CU(cudaMemcpyAsync(offall.data(), d_offall, offall.size() * 8, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  auto cnt = [&](int from, int to) { return offall[(size_t)from * (R + 1) + to + 1] - offall[(size_t)from * (R + 1) + to]; };
  u64 n_recv = 0, n_global = 0;
  std::vector<u64> roff(R + 1, 0);
  for (int q = 0; q < R; ++q) { roff[q] = n_recv; n_recv += cnt(q, rank); n_global += offall[(size_t)q * (R + 1) + R]; }
  roff[R] = n_recv;
  if (n_recv >= 0x7FFFFFFFull) return fail(ctx, CMX_ERR_INVALID, "cmx_dedup_shuffle: %llu records in this rank's key range exceed 2^31-1", (unsigned long long)n_recv);
  const u64 nr1 = std::max<u64>(n_recv, 1);
  CU(d_recv.alloc(nr1 * sizeof(PpRecord))); CU(d_res.alloc(nr1 * sizeof(PpRecord)));
  if (bc) { CU(d_recvbc.alloc(nr1 * 8)); CU(d_resbc.alloc(nr1 * 8)); }
  // ---- shuffle: every record travels once, to the rank that owns its key range
  CU(cudaEventRecord(ev[1], st));
  NC(N.GroupStart());
  for (int q = 0; q < R; ++q) {
    const u64 so = offall[(size_t)rank * (R + 1) + q], sc = cnt(rank, q), rc = cnt(q, rank);
    if (q == rank) {  // this rank's own share stays on the device
      if (sc) {
        CU(cudaMemcpyAsync(d_recv + roff[q], d_send + so, sc * sizeof(PpRecord), cudaMemcpyDeviceToDevice, st));
        if (bc) CU(cudaMemcpyAsync(d_recvbc + roff[q], d_sendbc + so, sc * 8, cudaMemcpyDeviceToDevice, st));
      }
      continue;
    }
    if (sc) {
      NC(N.Send(d_send + so, sc * sizeof(PpRecord), NCCL_UINT8, q, ctx->nccl_comm, st));
      if (bc) NC(N.Send(d_sendbc + so, sc * 8, NCCL_UINT8, q, ctx->nccl_comm, st));
    }
    if (rc) {
      NC(N.Recv(d_recv + roff[q], rc * sizeof(PpRecord), NCCL_UINT8, q, ctx->nccl_comm, st));
      if (bc) NC(N.Recv(d_recvbc + roff[q], rc * 8, NCCL_UINT8, q, ctx->nccl_comm, st));
    }
  }
  NC(N.GroupEnd());
  CU(cudaEventRecord(ev[2], st));
  // ---- the ordinary single-GPU post-processing of what arrived
  PpParams P;
  P.kind = bc ? PP_BED_BC : PP_BED; P.low_mem = 1; P.dedup = p.remove_pcr_duplicates; P.tn5 = p.tn5_shift; P.mapq_threshold = p.mapq_threshold; P.se = 0;
  u64 nsel = 0;
  const int prc = pp_device(ctx, P, d_recv, d_recvbc, n_recv, d_res, d_resbc, &nsel);
  if (prc != CMX_OK) return prc;
  CU(cudaEventRecord(ev[3], st));
  *n_out = nsel;
  if (nsel > out_capacity) return fail(ctx, CMX_ERR_INVALID, "cmx_dedup_shuffle: %llu records for a capacity of %llu", (unsigned long long)nsel, (unsigned long long)out_capacity);
  if (nsel) {
    const cudaMemcpyKind kind = on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
    CU(cudaMemcpyAsync(out_records, d_res, nsel * sizeof(PpRecord), kind, st));
    if (bc && out_barcode_keys) CU(cudaMemcpyAsync(out_barcode_keys, d_resbc, nsel * 8, kind, st));
  }
  CU(cudaStreamSynchronize(st));
  CU(cudaGetLastError());
  if (stats) {
    cudaEventElapsedTime(&stats->partition_ms, ev[0], ev[1]);
    cudaEventElapsedTime(&stats->shuffle_ms, ev[1], ev[2]);
    cudaEventElapsedTime(&stats->postprocess_ms, ev[2], ev[3]);
    const u64 rb = sizeof(PpRecord) + (bc ? 8 : 0);
    stats->bytes_sent = (n - cnt(rank, rank)) * rb; stats->bytes_received = (n_recv - cnt(rank, rank)) * rb;
    stats->n_received = n_recv; stats->n_global = n_global; stats->n_ranks = (uint32_t)R;
  }
  return CMX_OK;
}

// Last step after the survivors of all ranks have been brought together (e.g. on rank 0): reference order and the deferred
// Tn5 shift (mapping_writer.h:285-287).  Host only (no device needed), in place.
int cmx_exchange_finish(const cmx_params *params, cmx_pe_record *recs, uint64_t *bcs, uint64_t n) {
  if (!params || (!recs && n)) return CMX_ERR_INVALID;
  std::vector<u64> order(n);
  for (u64 i = 0; i < n; ++i) order[i] = i;
  auto key = [&](u64 i) { const cmx_pe_record &r = recs[i]; return std::make_tuple(r.rid, r.fragment_start, r.fragment_length, bcs ? bcs[i] : 0ull, r.mapq, r.direction, r.is_unique, r.read_id); };
  std::stable_sort(order.begin(), order.end(), [&](u64 x, u64 y) { return key(x) < key(y); });
  std::vector<cmx_pe_record> tmp(n);
  std::vector<u64> tb(bcs ? n : 0);
  for (u64 i = 0; i < n; ++i) { tmp[i] = recs[order[i]]; if (bcs) tb[i] = bcs[order[i]]; }
  for (u64 i = 0; i < n; ++i) { recs[i] = tmp[i]; if (bcs) bcs[i] = tb[i]; if (params->tn5_shift) tn5(recs[i]); }
  return CMX_OK;
}

// BED text on the device (bed_len_kernel / bed_write_kernel), byte-identical to cmx_format_bed / cmx_format_bed_bc.
// Records (and barcode keys, NULL for bulk data) and the output buffer are host memory; work goes through the device in
// chunks of 8 M records.  buf == NULL: returns the text length only.  Returns < 0 on error.
static int format_bed_gpu(cmx_ctx *ctx, const char *const *names, const cmx_pe_record *records, const uint64_t *barcode_keys, uint64_t n,
                          uint32_t bc_len, char *buf, int64_t cap, int64_t *total) {
  const u32 n_seq = ctx->n_seq;
  std::string cat;
  std::vector<u32> noff(n_seq + 1, 0);
  for (u32 i = 0; i < n_seq; ++i) { cat += names[i]; noff[i + 1] = (u32)cat.size(); }
  const u64 CH = 8u << 20;
  const u64 nc = std::min<u64>(n, CH);
  DevMem<char> d_names, d_out;
  DevMem<u32> d_noff, d_len;
  DevMem<PpRecord> d_rec;
  DevMem<u64> d_bc, d_off;
  DevMem<> d_tmp;
  size_t tmp_bytes = 0;
  cudaStream_t st = ctx->stream;
  CU(d_names.alloc(cat.size() + 1)); CU(d_noff.alloc((n_seq + 1) * 4));
  CU(cudaMemcpyAsync(d_names, cat.data(), cat.size(), cudaMemcpyHostToDevice, st)); CU(cudaMemcpyAsync(d_noff, noff.data(), (n_seq + 1) * 4, cudaMemcpyHostToDevice, st));
  if (nc == 0) { CU(cudaGetLastError()); return CMX_OK; }
  CU(d_rec.alloc(nc * sizeof(PpRecord))); CU(d_len.alloc((nc + 1) * 4)); CU(d_off.alloc((nc + 1) * 8));
  if (barcode_keys) CU(d_bc.alloc(nc * 8));
  cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, d_len.p, d_off.p, (int)nc + 1, st);
  CU(d_tmp.alloc(tmp_bytes));
  // --barcode-translate: every segment must have an entry before any text is written.  The length pass counts those that do
  // not; with more than one chunk, a first round of length passes checks the whole call before the round that writes.
  BedTranslation T{};
  DevMem<unsigned long long> d_miss;
  const bool tr = barcode_keys && ctx->tr_n_slots;
  if (tr) {
    CU(d_miss.alloc(16));
    const unsigned long long init[2] = {0ull, ~0ull};
    CU(cudaMemcpyAsync(d_miss, init, 16, cudaMemcpyHostToDevice, st));
    T.slots = ctx->tr_slots; T.mask = ctx->tr_n_slots - 1; T.shift = table_shift(ctx->tr_n_slots); T.from_len = (int)ctx->tr_from_len; T.to = ctx->tr_to;
    T.n_missing = d_miss.p; T.first_missing = reinterpret_cast<unsigned *>(d_miss.p + 1);  // (a chunk has < 2^32 records)
  }
  for (int round = tr && buf && n > CH ? 0 : 1; round < 2; ++round) {
    for (u64 c0 = 0; c0 < n; c0 += CH) {
      const u64 m = std::min(CH, n - c0);
      const unsigned nb = (unsigned)((m + 255) / 256);
      CU(cudaMemcpyAsync(d_rec, records + c0, m * sizeof(PpRecord), cudaMemcpyHostToDevice, st));
      if (barcode_keys) CU(cudaMemcpyAsync(d_bc, barcode_keys + c0, m * 8, cudaMemcpyHostToDevice, st));
      CU(cudaMemsetAsync(d_len + m, 0, 4, st));
      bed_len_kernel<<<nb, 256, 0, st>>>(d_rec, m, d_noff, barcode_keys ? (int)bc_len : 0, d_len, d_bc, T);
      CU(cub::DeviceScan::ExclusiveSum(d_tmp, tmp_bytes, d_len.p, d_off.p, (int)m + 1, st));
      u64 bytes = 0;
      unsigned long long miss[2] = {0ull, 0ull};
      CU(cudaMemcpyAsync(&bytes, d_off + m, 8, cudaMemcpyDeviceToHost, st));
      if (tr) CU(cudaMemcpyAsync(miss, d_miss, 16, cudaMemcpyDeviceToHost, st));
      CU(cudaStreamSynchronize(st));
      if (miss[0]) {  // the first chunk with a missing segment (the count covers the chunks so far, all of them without one)
        const u64 first = c0 + (u32)miss[1];
        std::string bc;
        for (u32 j = 0; j < bc_len; ++j) bc += "ACGT"[(barcode_keys[first] >> ((bc_len - 1 - j) * 2)) & 3];
        return fail(ctx, CMX_ERR_BARCODE_TRANSLATE, "%llu barcode segments have no entry in the translation table; the first is in barcode %s (record %llu)", miss[0],
                    bc.c_str(), (unsigned long long)first);
      }
      if (round == 1 && buf && *total + (int64_t)bytes <= cap) {
        if (bytes > d_out.cap) CU(d_out.alloc(bytes + bytes / 8));  // (alloc frees the smaller buffer first)
        bed_write_kernel<<<nb, 256, 0, st>>>(d_rec, d_bc, m, d_names, d_noff, barcode_keys ? (int)bc_len : 0, d_off, 0, d_out, T);
        CU(cudaMemcpyAsync(buf + *total, d_out, bytes, cudaMemcpyDeviceToHost, st)); CU(cudaStreamSynchronize(st));
      }
      if (round == 1) *total += (int64_t)bytes;
    }
  }
  CU(cudaGetLastError());
  return CMX_OK;
}
int64_t cmx_format_bed_gpu(cmx_ctx *ctx, const char *const *names, const cmx_pe_record *records, const uint64_t *barcode_keys, uint64_t n,
                           uint32_t bc_len, char *buf, int64_t cap) {
  if (!ctx || !names || (!records && n) || (barcode_keys && (bc_len == 0 || bc_len > 32))) return -1;
  if (cudaSetDevice(ctx->device) != cudaSuccess) return -1;
  int64_t total = 0;
  const int rc = format_bed_gpu(ctx, names, records, barcode_keys, n, bc_len, buf, cap, &total);
  return rc == CMX_OK ? total : rc == CMX_ERR_BARCODE_TRANSLATE ? rc : -1;
}

// Pairs text on the device (pairs_len_kernel / pairs_write_kernel), byte-identical to cmx_format_pairs: the header is
// written by the host, the lines by one thread each.  Read names travel as one concatenation + offsets.
static int format_pairs_gpu(cmx_ctx *ctx, const char *const *names, uint32_t n_seq, const cmx_pairs_record *records, uint64_t n,
                            const char *const *read_names, uint64_t n_read_names, uint32_t first_read_id, char *buf, int64_t cap, int64_t *total) {
  std::string cat;
  std::vector<u32> noff(n_seq + 1, 0);
  for (u32 i = 0; i < n_seq; ++i) { cat += names[i]; noff[i + 1] = (u32)cat.size(); }
  std::vector<u64> roff(n_read_names + 1, 0);
  for (u64 i = 0; i < n_read_names; ++i) roff[i + 1] = roff[i] + strlen(read_names[i]);
  std::string rcat;
  rcat.resize(roff[n_read_names]);
  for (u64 i = 0; i < n_read_names; ++i) memcpy(&rcat[roff[i]], read_names[i], roff[i + 1] - roff[i]);
  DevMem<char> d_names, d_rn, d_out;
  DevMem<u32> d_noff, d_len;
  DevMem<u64> d_roff, d_off;
  DevMem<PpRecord> d_rec;
  DevMem<> d_tmp;
  size_t tmp_bytes = 0;
  cudaStream_t st = ctx->stream;
  const u64 CH = 8u << 20;
  const u64 nc = std::min<u64>(n, CH);
  CU(d_names.alloc(cat.size() + 1)); CU(d_noff.alloc((n_seq + 1) * 4)); CU(d_rn.alloc(rcat.size() + 1));
  CU(d_roff.alloc((n_read_names + 1) * 8)); CU(d_rec.alloc(nc * sizeof(PpRecord))); CU(d_len.alloc((nc + 1) * 4)); CU(d_off.alloc((nc + 1) * 8));
  CU(cudaMemcpyAsync(d_names, cat.data(), cat.size(), cudaMemcpyHostToDevice, st)); CU(cudaMemcpyAsync(d_noff, noff.data(), (n_seq + 1) * 4, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(d_rn, rcat.data(), rcat.size(), cudaMemcpyHostToDevice, st)); CU(cudaMemcpyAsync(d_roff, roff.data(), (n_read_names + 1) * 8, cudaMemcpyHostToDevice, st));
  cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, d_len.p, d_off.p, (int)nc + 1, st);
  CU(d_tmp.alloc(tmp_bytes));
  for (u64 c0 = 0; c0 < n; c0 += CH) {
    const u64 m = std::min(CH, n - c0);
    const unsigned nb = (unsigned)((m + 255) / 256);
    CU(cudaMemcpyAsync(d_rec, records + c0, m * sizeof(PpRecord), cudaMemcpyHostToDevice, st)); CU(cudaMemsetAsync(d_len + m, 0, 4, st));
    pairs_len_kernel<<<nb, 256, 0, st>>>(d_rec, m, d_noff, d_roff, first_read_id, d_len);
    CU(cub::DeviceScan::ExclusiveSum(d_tmp, tmp_bytes, d_len.p, d_off.p, (int)m + 1, st));
    u64 bytes = 0;
    CU(cudaMemcpyAsync(&bytes, d_off + m, 8, cudaMemcpyDeviceToHost, st)); CU(cudaStreamSynchronize(st));
    if (buf && *total + (int64_t)bytes <= cap) {
      if (bytes > d_out.cap) CU(d_out.alloc(bytes + bytes / 8));  // (alloc frees the smaller buffer first)
      pairs_write_kernel<<<nb, 256, 0, st>>>(d_rec, m, d_names, d_noff, d_rn, d_roff, first_read_id, d_off, d_out);
      CU(cudaMemcpyAsync(buf + *total, d_out, bytes, cudaMemcpyDeviceToHost, st)); CU(cudaStreamSynchronize(st));
    }
    *total += (int64_t)bytes;
  }
  CU(cudaGetLastError());
  return CMX_OK;
}
int64_t cmx_format_pairs_gpu(cmx_ctx *ctx, const char *const *names, const uint32_t *lengths, uint32_t n_seq, const cmx_pairs_record *records, uint64_t n,
                             const char *const *read_names, uint64_t n_read_names, uint32_t first_read_id, char *buf, int64_t cap) {
  if (!ctx || !names || !lengths || (!records && n) || (!read_names && n)) return -1;
  if (cudaSetDevice(ctx->device) != cudaSuccess) return -1;
  std::string hdr = "## pairs format v1.0.0\n#shape: upper triangle\n";  // mapping_writer.cc:383-402
  for (uint32_t i = 0; i < n_seq; ++i) hdr += std::string("#chromsize: ") + names[i] + " " + std::to_string(lengths[i]) + "\n";
  hdr += "#columns: readID chrom1 pos1 chrom2 pos2 strand1 strand2 pair_type mapq1 mapq2\n";
  int64_t total = (int64_t)hdr.size();
  if (buf && total <= cap) memcpy(buf, hdr.data(), hdr.size());
  if (n == 0) return total;
  return format_pairs_gpu(ctx, names, n_seq, records, n, read_names, n_read_names, first_read_id, buf, cap, &total) == CMX_OK ? total : -1;
}

struct WidenU64 {
  __host__ __device__ u64 operator()(u32 x) const { return x; }
};
static_assert(std::is_same<std::iterator_traits<thrust::transform_iterator<WidenU64, const u32 *>>::value_type, u64>::value,
              "SAM text offsets are scanned in 64 bits");
// SAM text on the device (sam_text.cuh), byte-identical to cmx_format_sam_bc; the caller writes the @SQ header.  Cores, keys and
// the reads of the call stay resident; lines are sorted by stable LSD radix passes over their ids, resolved, compacted, measured
// and scanned over the whole call, then written in chunks of 1 M lines.  *text_err = -2 / -3 as the host twin returns them.
static int format_sam_gpu(cmx_ctx *ctx, const char *const *ref_names, uint32_t n_seq, const cmx_sam_record *records, const uint64_t *barcode_keys,
                          uint32_t bc_len, uint64_t n, const cmx_read_set *reads1, const cmx_read_set *reads2, uint32_t first_read_id, char *buf,
                          int64_t cap, int64_t *total, int *text_err) {
  if (!ctx->ref_seq || n_seq != ctx->n_seq) return fail(ctx, CMX_ERR_STATE, "cmx_format_sam_gpu: the reference of these names is not uploaded");
  const bool pe = reads2 != nullptr;
  const u64 n_lines = n * (pe ? 2 : 1);
  if (n_lines > 0x7FFFFFFFull) return fail(ctx, CMX_ERR_INVALID, "cmx_format_sam_gpu: more than 2^31-1 lines in one call");
  cudaStream_t st = ctx->stream;
  const unsigned nb = (unsigned)((n_lines + 255) / 256);
  DevMem<OutSam> d_cores;
  DevMem<u64> d_bc, d_k0, d_k1, d_small;
  DevMem<u32> d_i0, d_i1, d_rnoff;
  DevMem<u8> d_head, d_keep;
  DevMem<char> d_rnames, d_out;
  DevMem<> d_tmp;
  CU(d_cores.alloc(n * sizeof(OutSam))); CU(d_small.alloc(64));
  CU(cudaMemcpyAsync(d_cores, records, n * sizeof(OutSam), cudaMemcpyHostToDevice, st));
  if (barcode_keys) { CU(d_bc.alloc(n * 8)); CU(cudaMemcpyAsync(d_bc, barcode_keys, n * 8, cudaMemcpyHostToDevice, st)); }
  CU(d_k0.alloc((n_lines + 1) * 8)); CU(d_k1.alloc((n_lines + 1) * 8)); CU(d_i0.alloc(n_lines * 4)); CU(d_i1.alloc(n_lines * 4));
  CU(d_head.alloc(n_lines)); CU(d_keep.alloc(n_lines));
  // d_small: [0] largest key word 0, [1] err (overflowed cores, long CIGARs), [2] selected lines, [3] largest read index,
  // [4, 5] missing translation segments / the first line that has one
  CU(cudaMemsetAsync(d_small, 0, 64, st));
  u64 *const max0 = d_small.p, *const nsel = d_small.p + 2;
  int *const err = reinterpret_cast<int *>(d_small.p + 1);
  u32 *const max_ri = reinterpret_cast<u32 *>(d_small.p + 3);
  SamText T{};
  T.cores = d_cores; T.bcs = barcode_keys ? d_bc.p : nullptr; T.pe = pe; T.bc_len = (int)bc_len; T.first_read_id = first_read_id;
  T.ref = ctx->ref_seq; T.ref_off = ctx->ref_off;
  sam_expand_kernel<<<nb, 256, 0, st>>>(T, n_lines, d_i0, max0, err);
  sam_max_read_kernel<<<nb, 256, 0, st>>>(T, n_lines, max_ri);
  u64 small[4];
  CU(cudaMemcpyAsync(small, d_small, 32, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  CU(cudaGetLastError());
  if ((int)(small[1] & 0xFFFFFFFFu)) { *text_err = -2; return CMX_OK; }
  const u64 n_reads = (u64)(u32)small[3] + 1;
  if (n_reads > 0x7FFFFFFFull) return fail(ctx, CMX_ERR_INVALID, "cmx_format_sam_gpu: a core's read id is below first_read_id");
  // the reads of the call, and the reference names
  DevMem<char> d_seq[2], d_qual[2], d_names[2];
  DevMem<u64> d_off[2], d_noff[2];
  std::string cat;
  for (int mate = 0; mate < (pe ? 2 : 1); ++mate) {
    const cmx_read_set &rs = mate ? *reads2 : *reads1;
    if (!rs.names || !rs.seq || !rs.off) return fail(ctx, CMX_ERR_INVALID, "cmx_format_sam_gpu: read set without names, bases or offsets");
    const u64 bytes = rs.off[n_reads];
    std::vector<u64> noff(n_reads + 1, 0);
    cat.clear();
    for (u64 i = 0; i < n_reads; ++i) { cat += rs.names[i]; noff[i + 1] = cat.size(); }
    CU(d_seq[mate].alloc(bytes + 1)); CU(d_off[mate].alloc((n_reads + 1) * 8)); CU(d_names[mate].alloc(cat.size() + 1)); CU(d_noff[mate].alloc((n_reads + 1) * 8));
    CU(cudaMemcpyAsync(d_seq[mate], rs.seq, bytes, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(d_off[mate], rs.off, (n_reads + 1) * 8, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(d_names[mate], cat.data(), cat.size(), cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(d_noff[mate], noff.data(), (n_reads + 1) * 8, cudaMemcpyHostToDevice, st));
    if (rs.qual) { CU(d_qual[mate].alloc(bytes + 1)); CU(cudaMemcpyAsync(d_qual[mate], rs.qual, bytes, cudaMemcpyHostToDevice, st)); }
    CU(cudaStreamSynchronize(st));  // (cat is reused)
    T.r[mate] = SamReads{d_seq[mate], rs.qual ? d_qual[mate].p : nullptr, d_off[mate], d_names[mate], d_noff[mate]};
  }
  std::vector<u32> rnoff(n_seq + 1, 0);
  cat.clear();
  for (u32 i = 0; i < n_seq; ++i) { cat += ref_names[i]; rnoff[i + 1] = (u32)cat.size(); }
  CU(d_rnames.alloc(cat.size() + 1)); CU(d_rnoff.alloc((n_seq + 1) * 4));
  CU(cudaMemcpyAsync(d_rnames, cat.data(), cat.size(), cudaMemcpyHostToDevice, st)); CU(cudaMemcpyAsync(d_rnoff, rnoff.data(), (n_seq + 1) * 4, cudaMemcpyHostToDevice, st));
  T.ref_names = d_rnames; T.ref_name_off = d_rnoff;
  // order: least significant word first, every pass stable; the barcode word only for barcoded cores, the mate position only
  // for paired-end ones (single-end lines all have 0)
  cub::DoubleBuffer<u64> dk(d_k0, d_k1);
  cub::DoubleBuffer<u32> di(d_i0, d_i1);
  size_t tmp_bytes = 0, need = 0;
  const int nl = (int)n_lines;
  cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, dk, di, nl, 0, 64, st);
  cub::DeviceSelect::Flagged(nullptr, need, d_i0.p, d_keep.p, d_i1.p, nsel, nl, st);
  tmp_bytes = std::max(tmp_bytes, need);
  cub::DeviceScan::ExclusiveSum(nullptr, need, thrust::make_transform_iterator(static_cast<const u32 *>(d_i0.p), WidenU64()), d_k0.p, nl + 1, st);
  tmp_bytes = std::max(tmp_bytes, need);
  CU(d_tmp.alloc(tmp_bytes));
  int bits0 = 1;
  while (bits0 < 64 && (small[0] >> bits0)) ++bits0;
  for (int w = 3; w >= 0; --w) {
    if ((w == 1 && !barcode_keys) || (w == 2 && !pe)) continue;
    sam_key_kernel<<<nb, 256, 0, st>>>(T, w, di.Current(), n_lines, dk.Current());
    const int bits = w == 0 ? bits0 : w == 1 ? 2 * (int)bc_len : w == 2 ? 32 : 41;
    CU(cub::DeviceRadixSort::SortPairs(d_tmp, tmp_bytes, dk, di, nl, 0, bits, st));
  }
  const cmx_params &p = ctx->params;
  u32 *const idx = di.Current(), *const res = di.Alternate();
  sam_head_kernel<<<nb, 256, 0, st>>>(T, p.remove_pcr_duplicates, idx, n_lines, d_head);
  sam_resolve_kernel<<<nb, 256, 0, st>>>(T, p.low_memory_mode, p.mapq_threshold, idx, d_head, n_lines, res, d_keep);
  // the key buffers are free now: selected line ids and lengths in one, the text offsets in the other; NM over the ids
  u32 *const sel = reinterpret_cast<u32 *>(dk.Alternate()), *const len = sel + n_lines, *const nm = idx;
  u64 *const off = dk.Current();
  CU(cub::DeviceSelect::Flagged(d_tmp, tmp_bytes, res, d_keep.p, sel, nsel, nl, st));
  CU(cudaMemcpyAsync(&small[2], nsel, 8, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  const u64 m = small[2];
  BedTranslation Tr{};
  const bool tr = barcode_keys && ctx->tr_n_slots;
  unsigned long long *const miss = reinterpret_cast<unsigned long long *>(d_small.p + 4);
  if (tr) {
    const unsigned first_init = ~0u;
    CU(cudaMemcpyAsync(d_small.p + 5, &first_init, 4, cudaMemcpyHostToDevice, st));
    Tr.slots = ctx->tr_slots; Tr.mask = ctx->tr_n_slots - 1; Tr.shift = table_shift(ctx->tr_n_slots); Tr.from_len = (int)ctx->tr_from_len; Tr.to = ctx->tr_to;
    Tr.n_missing = miss; Tr.first_missing = reinterpret_cast<unsigned *>(d_small.p + 5);
  }
  CU(cudaMemsetAsync(len + m, 0, 4, st));
  if (m) sam_len_kernel<<<(unsigned)((m + 255) / 256), 256, 0, st>>>(T, sel, m, len, nm, err, Tr);
  // the lengths are 32-bit, the text of a call is not: the scan must add in 64 bits (CUB's accumulator is the input's type)
  CU(cub::DeviceScan::ExclusiveSum(d_tmp, tmp_bytes, thrust::make_transform_iterator(static_cast<const u32 *>(len), WidenU64()), off, (int)m + 1, st));
  u64 res_small[6];
  CU(cudaMemcpyAsync(res_small, d_small, 48, cudaMemcpyDeviceToHost, st));
  u64 bytes_all = 0;
  CU(cudaMemcpyAsync(&bytes_all, off + m, 8, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  CU(cudaGetLastError());
  if ((res_small[1] >> 32) != 0) { *text_err = -3; return CMX_OK; }
  if (tr && res_small[4]) {
    const u32 first_line = (u32)res_small[5];
    u32 l = 0;
    CU(cudaMemcpy(&l, sel + first_line, 4, cudaMemcpyDeviceToHost));
    const u64 key = barcode_keys[pe ? l >> 1 : l];
    std::string bc;
    for (u32 j = 0; j < bc_len; ++j) bc += "ACGT"[(key >> ((bc_len - 1 - j) * 2)) & 3];
    return fail(ctx, CMX_ERR_BARCODE_TRANSLATE, "%llu barcode segments have no entry in the translation table; the first is in barcode %s (SAM line %u)",
                (unsigned long long)res_small[4], bc.c_str(), first_line);
  }
  const u64 CH = 1u << 20;
  const bool fits = buf && *total + (int64_t)bytes_all <= cap;
  for (u64 c0 = 0; fits && c0 < m; c0 += CH) {
    const u64 k = std::min(CH, m - c0);
    u64 ends[2];
    CU(cudaMemcpyAsync(&ends[0], off + c0, 8, cudaMemcpyDeviceToHost, st)); CU(cudaMemcpyAsync(&ends[1], off + c0 + k, 8, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    const u64 bytes = ends[1] - ends[0];
    if (bytes > d_out.cap) CU(d_out.alloc(bytes + bytes / 8));  // (alloc frees the smaller buffer first)
    sam_write_kernel<<<(unsigned)((k * 32 + 255) / 256), 256, 0, st>>>(T, sel + c0, k, off + c0, ends[0], nm + c0, d_out, Tr);
    CU(cudaMemcpyAsync(buf + *total + ends[0], d_out, bytes, cudaMemcpyDeviceToHost, st)); CU(cudaStreamSynchronize(st));
  }
  *total += (int64_t)bytes_all;
  CU(cudaGetLastError());
  return CMX_OK;
}
int64_t cmx_format_sam_gpu(cmx_ctx *ctx, const char *const *ref_names, const uint32_t *ref_lengths, uint32_t n_seq, const cmx_sam_record *records,
                           const uint64_t *barcode_keys, uint32_t bc_len, uint64_t n, const cmx_read_set *reads1, const cmx_read_set *reads2,
                           uint32_t first_read_id, char *buf, int64_t cap) {
  if (!ctx || !ref_names || !ref_lengths || (!records && n) || !reads1 || (barcode_keys && (bc_len == 0 || bc_len > 32))) return -1;
  if (cudaSetDevice(ctx->device) != cudaSuccess) return -1;
  std::string hdr;  // mapping_writer.cc:312-321
  for (uint32_t i = 0; i < n_seq; ++i) hdr += std::string("@SQ\tSN:") + ref_names[i] + "\tLN:" + std::to_string(ref_lengths[i]) + "\n";
  int64_t total = (int64_t)hdr.size();
  if (buf && total <= cap) memcpy(buf, hdr.data(), hdr.size());
  if (n == 0) return total;
  int text_err = 0;
  const int rc = format_sam_gpu(ctx, ref_names, n_seq, records, barcode_keys, bc_len, n, reads1, reads2, first_read_id, buf, cap, &total, &text_err);
  if (rc == CMX_OK) return text_err ? text_err : total;
  return rc == CMX_ERR_BARCODE_TRANSLATE ? rc : -1;
}

// --TagAlign for paired-end records (mapping_writer.cc:84-110): one line per mate, the duplicate count on the second.
// (Single-end TagAlign lines are the BED lines, mapping_writer.cc:55-62.)
int64_t cmx_format_tagalign(const char *const *names, const cmx_pe_record *recs, uint64_t n, char *buf, int64_t cap) {
  int64_t len = 0;
  char line[2200];
  for (uint64_t i = 0; i < n; ++i) {
    const cmx_pe_record &r = recs[i];
    const uint32_t pos_end = r.fragment_start + r.positive_alignment_length, neg_end = r.fragment_start + r.fragment_length;
    const uint32_t neg_start = neg_end - r.negative_alignment_length;
    const char *nm = names[r.rid];
    int l;
    if (r.direction)
      l = snprintf(line, sizeof(line), "%s\t%u\t%u\tN\t%u\t+\n%s\t%u\t%u\tN\t%u\t-\t%u\n", nm, r.fragment_start, pos_end, (uint32_t)r.mapq, nm, neg_start, neg_end,
                   (uint32_t)r.mapq, (uint32_t)r.num_dups);
    else
      l = snprintf(line, sizeof(line), "%s\t%u\t%u\tN\t%u\t-\n%s\t%u\t%u\tN\t%u\t+\t%u\n", nm, neg_start, neg_end, (uint32_t)r.mapq, nm, r.fragment_start, pos_end,
                   (uint32_t)r.mapq, (uint32_t)r.num_dups);
    if (buf && len + l <= cap) memcpy(buf + len, line, l);
    len += l;
  }
  return len;
}

int64_t cmx_format_bed(const char *const *names, const cmx_pe_record *recs, uint64_t n, char *buf, int64_t cap) {
  int64_t len = 0;
  char line[1100];
  for (uint64_t i = 0; i < n; ++i) {  // mapping_writer.cc:75-83
    const cmx_pe_record &r = recs[i];
    const int l = snprintf(line, sizeof(line), "%s\t%u\t%u\tN\t%u\t%c\t%u\n", names[r.rid], r.fragment_start,
                           (uint32_t)(r.fragment_start + r.fragment_length), (uint32_t)r.mapq, r.direction ? '+' : '-', (uint32_t)r.num_dups);
    if (buf && len + l <= cap) memcpy(buf + len, line, l);
    len += l;
  }
  return len;
}

}  // extern "C"
