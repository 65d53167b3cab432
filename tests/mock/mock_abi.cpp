// CPU stand-in for librg_b200.so, TEST INFRASTRUCTURE ONLY (tests/test_driver_plumbing_cpu.py).
//
// It implements the entry points of include/rg_b200.h that the rgb200 driver calls, with small, deterministic,
// data-dependent arithmetic that has nothing to do with regenie's statistics: every output is a simple function of the
// bytes and numbers the driver handed over (genotype rows, residuals, masks, W slabs).  Linked with the driver's own
// sources into `rgb200_mock`, it lets the CPU suite run the driver's control flow end to end - option handling, file
// readers and writers, block prefetch, --split-l0 / --run-l0 / --run-l1 files, --chr / --range jobs, .gz and PRS paths,
// --gpu-inflate buffers, Firth / SPA selection - and check the equivalences the reference's own tests check (sharded ==
// unsharded, window == subset of the full run, compressed == plain) where no GPU exists.  Nothing here is shipped,
// measured or compared with the reference's numbers; the product library never links it.
#include <zlib.h>

#include <cmath>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/rg_b200.h"
#include "../../regenie_b200/csrc/pgen_core.h"

struct rg_ctx {
  int kind = 0;
  int64_t N = 0;
  int P = 0, C = 0, K = 0, R = 0, R1 = 0, nb = 0, bs_max = 0;
  std::vector<double> Y, res, scf;
  std::vector<uint8_t> mask, in_analysis, l1_sel, male, nonpar;
  std::map<std::pair<int, int>, std::vector<double>> W;        // (block, pheno) -> N x R slab of the phenotypes owned here
  std::vector<rg_ctx*> W_owner;                                // per pheno: the handle whose W holds it (rg_W_attach_local)
  std::vector<double> prs;
  std::vector<double> last_stat;                               // [bs x P] of the last block (Firth / SPA)
  std::vector<uint8_t> inflate_probs, inflate_miss;
  std::vector<uint32_t> pgen_rows;
  std::vector<uint8_t> stage[4];                               // rg_s2_stage slots (host copies)
  int last_bs = 0;
  int ordinal = 0;                                             // creation order of the handles, from 1 (RG_MOCK_TRACE)
  bool qt_chr = false, bt_chr = false;                         // rg_s2_set_chr / rg_s2_set_chr_bt has run
};

namespace {
thread_local std::string g_err;                               // one driver thread per device: errors stay with their thread
std::mutex g_W_mu;                                            // level-0 slabs of a phenotype land in its owner's W
int fail(const std::string& m) { g_err = m; return 1; }

// RG_MOCK_TRACE=<file>: one line per Step-2 entry point - its name, the handle's creation ordinal, bs or n_sel, min_mac, the
// non-PAR flags pending on the handle, and for the set_* calls a checksum of the bytes uploaded - so that a driver change
// can be checked for the calls it makes, their order and their handle, which the output files alone do not show
std::mutex g_trace_mu;
int g_handles = 0;
uint64_t fnv(const void* p, size_t n, uint64_t s = 1469598103934665603ull) {
  for (size_t i = 0; i < n; ++i) s = (s ^ ((const uint8_t*)p)[i]) * 1099511628211ull;
  return s;
}
void trace(const char* name, const rg_ctx* h, long n, double min_mac = -1, uint64_t sum = 0) {
  static const char* path = getenv("RG_MOCK_TRACE");
  if (!path) return;
  std::lock_guard<std::mutex> lk(g_trace_mu);
  if (FILE* f = fopen(path, "a")) {                           // opened per line: the driver leaves through _exit
    fprintf(f, "%s %d %ld %g %zu %016llx\n", name, h ? h->ordinal : 0, n, min_mac, h ? h->nonpar.size() : 0, (unsigned long long)sum);
    fclose(f);
  }
}

// PLINK 1 code -> ALT-allele count as the driver's kernels see it (ref-last): 00 -> 2, 01 -> missing, 10 -> 1, 11 -> 0
inline int bed_call(const uint8_t* row, int64_t s) {
  const int code = (row[s >> 2] >> (2 * (s & 3))) & 3;
  return code == 0 ? 2 : code == 1 ? -1 : code == 2 ? 1 : 0;
}

struct Geno { std::vector<double> g; std::vector<uint8_t> miss; };

// genotype of every kept sample for one variant
Geno from_bed(const rg_ctx* h, const uint8_t* row, const int32_t* sample_idx, int ref_first) {
  Geno o; o.g.resize(h->N); o.miss.resize(h->N);
  for (int64_t s = 0; s < h->N; ++s) {
    const int c = bed_call(row, sample_idx ? sample_idx[s] : s);
    o.miss[s] = c < 0;
    o.g[s] = c < 0 ? 0.0 : (ref_first ? 2 - c : c);
  }
  return o;
}
Geno from_bgen(const rg_ctx* h, const uint8_t* probs, const uint8_t* pm, const int32_t* sample_idx, int ref_first) {
  Geno o; o.g.resize(h->N); o.miss.resize(h->N);
  for (int64_t s = 0; s < h->N; ++s) {
    const int64_t f = sample_idx ? sample_idx[s] : s;
    const double a = probs[2 * f] / 255.0, b = probs[2 * f + 1] / 255.0;
    o.miss[s] = pm && (pm[f] & 0x80);
    const double d = ref_first ? b + 2 * std::max(1 - a - b, 0.0) : b + 2 * a;
    o.g[s] = o.miss[s] ? 0.0 : d;
  }
  return o;
}

// the mock "test": per trait, counts and a correlation-like statistic with the residuals the driver uploaded
void score(rg_ctx* h, int v, const Geno& x, const std::vector<double>& res, double min_mac, const rg_s2_out* o, double* info) {
  const int P = h->P;
  const int64_t N = h->N;
  double tot = 0; int64_t ns_all = 0;
  for (int64_t s = 0; s < N; ++s) if (h->in_analysis[s] && !x.miss[s]) { tot += x.g[s]; ++ns_all; }
  o->af_all[v] = ns_all ? tot / (2.0 * ns_all) : 0;
  o->ns_all[v] = (int32_t)ns_all;
  o->mac_all[v] = std::min(tot, 2.0 * ns_all - tot);
  const bool non_par = !h->nonpar.empty() && v < (int)h->nonpar.size() && h->nonpar[v];
  o->flags[v] = 0;
  o->scale_fac[v] = 1.0;
  bool any = false;
  for (int i = 0; i < P; ++i) {
    double sg = 0, sgg = 0, num = 0, males = 0; int64_t ns = 0;
    for (int64_t s = 0; s < N; ++s) {
      if (!h->mask[(size_t)i * N + s] || x.miss[s]) continue;
      sg += x.g[s]; sgg += x.g[s] * x.g[s]; ++ns;
      num += x.g[s] * res[(size_t)i * N + s];
      if (non_par && !h->male.empty() && h->male[s]) males += 1;
    }
    const size_t e = (size_t)v * P + i;
    o->af[e] = ns ? sg / (2.0 * ns) : 0;
    o->ns[e] = (int32_t)ns;
    o->mac[e] = std::min(sg, 2.0 * ns - males - sg);
    const double den = std::sqrt(sgg - (ns ? sg * sg / ns : 0) + 1e-3);
    o->stat[e] = num / den;
    o->beta[e] = o->stat[e] * (h->scf.empty() ? 1.0 : h->scf[i]) / den;
    o->se[e] = std::fabs(o->beta[e] / (o->stat[e] == 0 ? 1.0 : o->stat[e]));
    o->chisq[e] = o->stat[e] * o->stat[e];
    if (info) info[e] = std::min(1.0, 0.5 + sgg / (4.0 * ns + 1.0));
    any |= o->mac[e] >= min_mac;
    h->last_stat[e] = o->stat[e];
  }
  if (!any) o->flags[v] |= 1;
}
}  // namespace

extern "C" {

const char* rg_last_error(void) { return g_err.c_str(); }
const char* rg_version(void) { return "mock ABI for host-plumbing tests"; }
int rg_device_count(void) {
  const char* e = getenv("RG_MOCK_DEVICES");
  return e ? atoi(e) : 1;
}
int rg_warmup(int32_t) { return 0; }
int rg_l0_wait_input(rg_handle) { return 0; }
void rg_destroy(rg_handle h) { delete h; }
int rg_sync(rg_handle) { return 0; }

// ------------------------------------------------------------------ step 1
int rg_step1_create(const rg_step1_config* cfg, const double*, const double* Y, const uint8_t* mask, const uint8_t* in_analysis,
                    const int64_t*, const double*, const double*, rg_handle* out) {
  rg_ctx* h = new rg_ctx;
  h->ordinal = ++g_handles;
  h->kind = 1; h->N = cfg->n_samples; h->P = cfg->n_pheno; h->C = cfg->n_cov; h->K = cfg->n_folds; h->R = cfg->n_ridge_l0;
  h->R1 = cfg->n_ridge_l1; h->nb = cfg->total_blocks; h->bs_max = cfg->max_block_size;
  h->Y.assign(Y, Y + (size_t)h->N * h->P);
  h->mask.assign(mask, mask + (size_t)h->N * h->P);
  h->in_analysis.assign(in_analysis, in_analysis + h->N);
  h->l1_sel.assign(h->P, 1);
  h->W_owner.assign(h->P, h);
  *out = h;
  return 0;
}

// the slab of (block, pheno): column r, sample s = mean genotype-weighted phenotype, a function of every input byte; it is
// stored in the W of the phenotype's owner, like the library's peer stores
static void store_W(rg_handle h, int block_id, int bs, const std::vector<double>& colsum) {
  for (int p = 0; p < h->P; ++p) {
    std::vector<double> w((size_t)h->N * h->R, 0.0);
    for (int r = 0; r < h->R; ++r)
      for (int64_t s = 0; s < h->N; ++s)
        w[(size_t)r * h->N + s] = h->mask[(size_t)p * h->N + s] ? (colsum[s] / bs - 1.0) * (r + 1) * 0.1 + 0.01 * h->Y[(size_t)p * h->N + s] : 0.0;
    std::lock_guard<std::mutex> lk(g_W_mu);
    h->W_owner[p]->W[{block_id, p}] = std::move(w);
  }
}

int rg_l0_block_bed(rg_handle h, const uint8_t* packed, int64_t row_stride, int32_t bs, const int32_t* sample_idx, int32_t ref_first,
                    int32_t block_id) {
  if (block_id < 0 || block_id >= h->nb || bs > h->bs_max) return fail("mock: bad block");
  std::vector<double> colsum(h->N, 0.0);
  for (int v = 0; v < bs; ++v) {
    const Geno x = from_bed(h, packed + (size_t)v * row_stride, sample_idx, ref_first);
    for (int64_t s = 0; s < h->N; ++s) colsum[s] += (x.g[s] + 0.25 * x.miss[s]) * (1.0 + 0.001 * (v % 17));
  }
  store_W(h, block_id, bs, colsum);
  return 0;
}
int rg_l0_block_dosage_u8(rg_handle h, const uint8_t* probs, const uint8_t* pm, int64_t n_file, int32_t bs, const int32_t* sample_idx,
                          int32_t ref_first, int32_t block_id) {
  if (block_id < 0 || block_id >= h->nb || bs > h->bs_max) return fail("mock: bad block");
  // same deterministic function of the inputs as rg_l0_block_bed, on dosage units of 1/255
  std::vector<double> colsum(h->N, 0.0);
  for (int v = 0; v < bs; ++v)
    for (int64_t s = 0; s < h->N; ++s) {
      const int64_t f = sample_idx ? sample_idx[s] : s;
      const uint8_t* pr = probs + ((size_t)v * n_file + f) * 2;
      const bool miss = pm && (pm[(size_t)v * n_file + f] & 0x80);
      const double g = miss ? 0.25 : (ref_first ? 2.0 - (2.0 * pr[0] + pr[1]) / 255.0 : (2.0 * pr[0] + pr[1]) / 255.0);
      colsum[s] += g * (1.0 + 0.001 * (v % 17));
    }
  store_W(h, block_id, bs, colsum);
  return 0;
}
int64_t rg_l0_status(rg_handle) { return 0; }
int64_t rg_l0_poll_status(rg_handle) { return 0; }
int rg_l0_fetch_W(rg_handle h, int32_t b, int32_t ph, double* out) {
  auto it = h->W.find({b, ph});
  if (it == h->W.end()) return fail("mock: slab not computed");
  memcpy(out, it->second.data(), it->second.size() * 8);
  return 0;
}
int rg_l0_load_W(rg_handle h, int32_t b, int32_t ph, const double* in) {
  h->W[{b, ph}].assign(in, in + (size_t)h->N * h->R);
  return 0;
}
// --gpus N (RG_MOCK_DEVICES handles): level 1 runs on the owned phenotypes (rg_api.cu rg_W_set_owned), and the level-0
// slabs of a phenotype owned by a peer go to the peer's W map
int rg_W_set_owned(rg_handle h, const uint8_t* owned) {
  if (!h || !owned || !h->W.empty()) return fail("mock: rg_W_set_owned must come before the first block");
  for (int p = 0; p < h->P; ++p) h->l1_sel[p] = owned[p] ? 1 : 0;
  return 0;
}
int rg_W_attach_local(rg_handle h, rg_handle peer, const uint8_t* owned_by_peer) {
  if (!h || !peer || peer == h || !owned_by_peer) return fail("mock: bad rg_W_attach_local arguments");
  for (int p = 0; p < h->P; ++p) if (owned_by_peer[p]) h->W_owner[p] = peer;
  return 0;
}
int rg_l1_select(rg_handle h, const uint8_t* sel) { h->l1_sel.assign(sel, sel + h->P); return 0; }

static int l1_common(rg_handle h, const double* tau, double* cs, int32_t* best, int nsums) {
  for (int p = 0; p < h->P; ++p) {
    best[p] = 0;
    if (!h->l1_sel[p]) continue;
    double wsum = 0;
    for (int b = 0; b < h->nb; ++b) {
      auto it = h->W.find({b, p});
      if (it == h->W.end()) return fail("mock: level 1 without the level-0 slab of block " + std::to_string(b));
      for (double v : it->second) wsum += v * v;
    }
    double bestv = 1e300;
    for (int j = 0; j < h->R1; ++j) {
      const double t = tau[(size_t)p * h->R1 + j], f = wsum / (wsum + t * 1e-4);
      const double sx = 0.1 * f, sy = 0.2, sx2 = 10 * f * f + 1, sy2 = 12, sxy = 5 * f;
      const double v[6] = {sx, sy, sx2, sy2, sxy, 100 * (1 - f) + std::fabs(j - 2.0)};
      for (int k = 0; k < nsums; ++k) cs[((size_t)k * h->P + p) * h->R1 + j] = v[k];
      const double perf = nsums == 6 ? v[5] : sx2 + sy2 - 2 * sxy;
      if (perf < bestv) { bestv = perf; best[p] = j; }
    }
  }
  return 0;
}
int rg_l1_fit(rg_handle h, const double* tau, double* cs, int32_t* best) { return l1_common(h, tau, cs, best, 5); }
int rg_l1_fit_bt(rg_handle h, const double*, const double*, const double* tau, double* cs, int32_t* best) {
  return l1_common(h, tau, cs, best, 6);
}
int rg_loco(rg_handle h, const int32_t* chr_of_block, double* out) {
  const int64_t N = h->N;
  h->prs.assign((size_t)h->P * N, 0.0);
  for (int p = 0; p < h->P; ++p) {
    if (!h->l1_sel[p]) continue;
    std::vector<double> per_chr((size_t)23 * N, 0.0), tot(N, 0.0);
    for (int b = 0; b < h->nb; ++b) {
      const std::vector<double>& w = h->W[{b, p}];
      for (int64_t s = 0; s < N; ++s) {
        double v = 0;
        for (int r = 0; r < h->R; ++r) v += 0.02 * w[(size_t)r * N + s] / (r + 2.0);   // small, like real polygenic predictions
        per_chr[(size_t)(chr_of_block[b] - 1) * N + s] += v;
        tot[s] += v;
      }
    }
    for (int c = 0; c < 23; ++c)
      for (int64_t s = 0; s < N; ++s) out[((size_t)p * 23 + c) * N + s] = tot[s] - per_chr[(size_t)c * N + s];
    for (int64_t s = 0; s < N; ++s) h->prs[(size_t)p * N + s] = tot[s];
  }
  return 0;
}
int rg_prs(rg_handle h, double* out) {
  if (h->prs.empty()) return fail("mock: rg_loco first");
  memcpy(out, h->prs.data(), h->prs.size() * 8);
  return 0;
}

// ------------------------------------------------------------------ step 2
int rg_step2_create(const rg_step2_config* cfg, const double*, const uint8_t* mask, const uint8_t* in_analysis, rg_handle* out) {
  rg_ctx* h = new rg_ctx;
  h->ordinal = ++g_handles;
  h->kind = 2; h->N = cfg->n_samples; h->P = cfg->n_pheno; h->C = cfg->n_cov; h->bs_max = cfg->max_block_size;
  h->mask.assign(mask, mask + (size_t)h->N * h->P);
  h->in_analysis.assign(in_analysis, in_analysis + h->N);
  h->last_stat.assign((size_t)h->bs_max * h->P, 0.0);
  trace("rg_step2_create", h, h->bs_max, -1, fnv(mask, (size_t)h->N * h->P));
  *out = h;
  return 0;
}
int rg_s2_set_chr(rg_handle h, const double* res, const double* scf) {
  trace("rg_s2_set_chr", h, 0, -1, fnv(scf, (size_t)h->P * 8, fnv(res, (size_t)h->N * h->P * 8)));
  h->res.assign(res, res + (size_t)h->N * h->P);
  h->scf.assign(scf, scf + h->P);
  h->qt_chr = true;
  return 0;
}
int rg_s2_set_sex(rg_handle h, const uint8_t* male) {
  trace("rg_s2_set_sex", h, male ? h->N : 0, -1, male ? fnv(male, h->N) : 0);
  if (male) h->male.assign(male, male + h->N); else h->male.clear();
  return 0;
}
int rg_s2_set_non_par(rg_handle h, const uint8_t* flags, int32_t n) {
  trace("rg_s2_set_non_par", h, n, -1, fnv(flags, n));
  h->nonpar.assign(flags, flags + n);
  return 0;
}
int rg_s2_set_chr_bt(rg_handle h, const rg_s2_bt_chr* st) {
  const size_t NP = (size_t)h->N * h->P * 8;
  uint64_t sum = fnv(st->yres, NP, fnv(st->gamma_sqrt, NP, fnv(st->gamma_sqrt_mask, NP)));
  sum = fnv(st->y_raw, NP, fnv(st->x_gamma, NP * h->C, sum));
  if (st->firth_offset) sum = fnv(st->firth_offset, NP, sum);
  if (st->y_hat_p) sum = fnv(st->y_hat_p, NP, sum);
  trace("rg_s2_set_chr_bt", h, 0, -1, sum);
  h->res.assign(st->yres, st->yres + (size_t)h->N * h->P);
  for (size_t e = 0; e < h->res.size(); ++e) h->res[e] *= 25.0 * st->gamma_sqrt_mask[e];   // enough |z| > threshold cases
  h->scf.assign(h->P, 1.0);
  h->bt_chr = true;
  return 0;
}
// each route needs its own chromosome call, like the library: a driver that calls the route of the other trait kind fails
static int block_common(rg_handle h, bool bt, int bs) {
  if (h->kind != 2 || bs < 1 || bs > h->bs_max) return fail("mock: block size out of range");
  if (!(bt ? h->bt_chr : h->qt_chr)) return fail(bt ? "mock: rg_s2_set_chr_bt has not been called" : "mock: rg_s2_set_chr has not been called");
  h->last_bs = bs;
  return 0;
}
static int block_bed(rg_handle h, bool bt, const uint8_t* packed, int64_t row_stride, int32_t bs, const int32_t* sample_idx,
                     int32_t ref_first, double min_mac, const rg_s2_out* o) {
  if (block_common(h, bt, bs)) return 1;
  for (int v = 0; v < bs; ++v) score(h, v, from_bed(h, packed + (size_t)v * row_stride, sample_idx, ref_first), h->res, min_mac, o, nullptr);
  h->nonpar.clear();
  return 0;
}
static int block_bgen8(rg_handle h, bool bt, const uint8_t* probs, const uint8_t* pm, int64_t n_file, int32_t bs, const int32_t* sample_idx,
                       int32_t ref_first, double min_mac, const rg_s2_out* o, double* info) {
  if (block_common(h, bt, bs)) return 1;
  for (int v = 0; v < bs; ++v)
    score(h, v, from_bgen(h, probs + (size_t)v * n_file * 2, pm ? pm + (size_t)v * n_file : nullptr, sample_idx, ref_first), h->res,
          min_mac, o, info);
  h->nonpar.clear();
  return 0;
}
int rg_s2_block_bed(rg_handle h, const uint8_t* packed, int64_t row_stride, int32_t bs, const int32_t* sample_idx, int32_t ref_first,
                    double min_mac, const rg_s2_out* o) {
  trace("rg_s2_block_bed", h, bs, min_mac);
  return block_bed(h, false, packed, row_stride, bs, sample_idx, ref_first, min_mac, o);
}
int rg_s2_block_bed_bt(rg_handle h, const uint8_t* packed, int64_t row_stride, int32_t bs, const int32_t* sample_idx, int32_t ref_first,
                       double min_mac, const rg_s2_out* o) {
  trace("rg_s2_block_bed_bt", h, bs, min_mac);
  return block_bed(h, true, packed, row_stride, bs, sample_idx, ref_first, min_mac, o);
}
int rg_s2_block_bgen8(rg_handle h, const uint8_t* probs, const uint8_t* pm, int64_t n_file, int32_t bs, const int32_t* sample_idx,
                      int32_t ref_first, double min_mac, const rg_s2_out* o, double* info) {
  trace("rg_s2_block_bgen8", h, bs, min_mac);
  return block_bgen8(h, false, probs, pm, n_file, bs, sample_idx, ref_first, min_mac, o, info);
}
int rg_s2_block_bgen8_bt(rg_handle h, const uint8_t* probs, const uint8_t* pm, int64_t n_file, int32_t bs, const int32_t* sample_idx,
                         int32_t ref_first, double min_mac, const rg_s2_out* o, double* info) {
  trace("rg_s2_block_bgen8_bt", h, bs, min_mac);
  return block_bgen8(h, true, probs, pm, n_file, bs, sample_idx, ref_first, min_mac, o, info);
}
int rg_s2_firth(rg_handle h, int32_t n, const int32_t* vi, const int32_t* ti, double* beta, double* se, double* lrt, int32_t* status) {
  trace("rg_s2_firth", h, n);
  for (int k = 0; k < n; ++k) {
    if (vi[k] < 0 || vi[k] >= h->last_bs || ti[k] < 0 || ti[k] >= h->P) return fail("mock: bad Firth selection");
    const double z = h->last_stat[(size_t)vi[k] * h->P + ti[k]];
    beta[k] = 0.9 * z; se[k] = 0.9; lrt[k] = 0.81 * z * z;
    status[k] = (vi[k] % 5 == 2) ? 1 : 0;                    // some failures -> TEST_FAIL rows
  }
  return 0;
}
int rg_s2_spa(rg_handle h, int32_t n, const int32_t* vi, const int32_t* ti, double* pval, int32_t* status) {
  trace("rg_s2_spa", h, n);
  for (int k = 0; k < n; ++k) {
    if (vi[k] < 0 || vi[k] >= h->last_bs || ti[k] < 0 || ti[k] >= h->P) return fail("mock: bad SPA selection");
    pval[k] = std::erfc(std::fabs(h->last_stat[(size_t)vi[k] * h->P + ti[k]]) * 0.6);
    status[k] = 0;
  }
  return 0;
}
// zlib on the host: the mock's block entry points take host pointers
int rg_bgen_inflate(rg_handle h, const uint8_t* comp, const uint64_t* offs, int64_t n_file, int32_t bs, const uint8_t** probs,
                    const uint8_t** miss) {
  trace("rg_bgen_inflate", h, bs);
  h->inflate_probs.resize((size_t)bs * n_file * 2);
  h->inflate_miss.resize((size_t)bs * n_file);
  std::vector<uint8_t> raw(10 + 3 * (size_t)n_file);
  for (int v = 0; v < bs; ++v) {
    uLongf dl = raw.size();
    if (uncompress(raw.data(), &dl, comp + offs[v], (uLong)(offs[v + 1] - offs[v])) != Z_OK || dl != raw.size())
      return fail("mock: corrupt zlib stream");
    memcpy(&h->inflate_miss[(size_t)v * n_file], raw.data() + 8, (size_t)n_file);
    memcpy(&h->inflate_probs[(size_t)v * n_file * 2], raw.data() + 10 + n_file, (size_t)n_file * 2);
  }
  *probs = h->inflate_probs.data();
  *miss = h->inflate_miss.data();
  return 0;
}

// the device decoder's arithmetic (csrc/pgen_core.h), lanes run serially; rows live in the handle like the device buffer
int rg_pgen_decode(rg_handle h, const rg_pgen_block* b, const uint8_t** rows_dev, int64_t* row_stride) {
  if (!h || !b || !rows_dev || !row_stride || !b->bytes || b->bs <= 0 || b->n_file <= 0) return fail("mock: bad pgen block");
  trace("rg_pgen_decode", h, b->bs);
  const uint32_t n = (uint32_t)b->n_file, words = ((n + 15) / 16 + 3) / 4 * 4;
  h->pgen_rows.assign((size_t)b->bs * words, 0u);
  for (int j = 0; j < b->bs; ++j) {
    auto rec = [&](int32_t r) { return rgp::Rec{b->bytes + b->rec_off[r], b->rec_len[r], b->rec_type[r]}; };
    if (b->own[j] < 0 || b->own[j] >= b->n_rec || b->base[j] >= b->n_rec) return fail("mock: pgen record index out of range");
    const rgp::Rec own = rec(b->own[j]);
    rgp::Rec base{nullptr, 0, 0};
    if (b->base[j] >= 0) base = rec(b->base[j]);
    if (rgp::decode_row_serial(own, b->base[j] >= 0 ? &base : nullptr, n, &h->pgen_rows[(size_t)j * words], words, 32))
      return fail("mock: malformed .pgen record");
  }
  *rows_dev = reinterpret_cast<const uint8_t*>(h->pgen_rows.data());
  *row_stride = (int64_t)words * 4;
  return 0;
}

// staging: a plain copy into the slot (what the block call later reads is the bytes as they were when staged)
int rg_s2_stage(rg_handle h, int32_t slot, const void* host, int64_t bytes, const uint8_t** dev) {
  if (!h || !host || !dev || bytes <= 0 || slot < 0 || slot > 3) return fail("mock: bad staging arguments");
  trace("rg_s2_stage", h, (long)bytes, -1, fnv(host, (size_t)bytes));
  h->stage[slot].assign((const uint8_t*)host, (const uint8_t*)host + bytes);
  *dev = h->stage[slot].data();
  return 0;
}
int rg_host_alloc(void** p, int64_t bytes) { *p = malloc((size_t)bytes); return *p ? 0 : fail("mock: out of memory"); }
int rg_host_free(void* p) { free(p); return 0; }

}  // extern "C"
