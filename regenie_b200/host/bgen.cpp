#include "bgen.hpp"
#include "textio.hpp"

#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>
#include <zlib.h>

#include <dlfcn.h>

#include <algorithm>
#include <atomic>
#include <cstring>
#include <thread>

namespace rgh {

namespace {
// zstd payloads (BGEN compression flag 2; the reference links BGEN's bundled zstd, src/Geno.cpp:1610, :2209).  Only the
// runtime library ships in this image, so the one entry point needed is bound with dlopen; lossless, no parity risk.
typedef size_t (*ZstdDecompressFn)(void*, size_t, const void*, size_t);
typedef unsigned (*ZstdIsErrorFn)(size_t);
ZstdDecompressFn g_zstd_decompress = nullptr;
ZstdIsErrorFn g_zstd_is_error = nullptr;
void load_zstd() {
  if (g_zstd_decompress) return;
  void* lib = dlopen("libzstd.so.1", RTLD_NOW);
  if (!lib) lib = dlopen("libzstd.so", RTLD_NOW);
  if (!lib) throw Fail("the bgen file is zstd-compressed but libzstd could not be loaded on this host.");
  g_zstd_decompress = reinterpret_cast<ZstdDecompressFn>(dlsym(lib, "ZSTD_decompress"));
  g_zstd_is_error = reinterpret_cast<ZstdIsErrorFn>(dlsym(lib, "ZSTD_isError"));
  if (!g_zstd_decompress || !g_zstd_is_error) throw Fail("libzstd does not export ZSTD_decompress.");
}

// .bgi index files are SQLite databases (bgenix); the reference reads them through its bundled sqlite3
// (read_bgi_file, src/Geno.cpp:180-309).  Only the runtime library ships in this image, so the handful of entry points
// is bound with dlopen, like zstd above.
struct Sqlite {
  typedef int (*OpenFn)(const char*, void**, int, const char*);
  typedef int (*PrepareFn)(void*, const char*, int, void**, const char**);
  typedef int (*StepFn)(void*);
  typedef const unsigned char* (*TextFn)(void*, int);
  typedef long long (*Int64Fn)(void*, int);
  typedef int (*FinalizeFn)(void*);
  typedef int (*CloseFn)(void*);
  typedef const char* (*ErrFn)(void*);
  OpenFn open = nullptr;
  PrepareFn prepare = nullptr;
  StepFn step = nullptr;
  TextFn text = nullptr;
  Int64Fn int64 = nullptr;
  FinalizeFn finalize = nullptr;
  CloseFn close = nullptr;
  ErrFn errmsg = nullptr;
  bool load() {
    if (open) return true;
    void* lib = dlopen("libsqlite3.so.0", RTLD_NOW);
    if (!lib) lib = dlopen("libsqlite3.so", RTLD_NOW);
    if (!lib) return false;
    open = reinterpret_cast<OpenFn>(dlsym(lib, "sqlite3_open_v2"));
    prepare = reinterpret_cast<PrepareFn>(dlsym(lib, "sqlite3_prepare_v2"));
    step = reinterpret_cast<StepFn>(dlsym(lib, "sqlite3_step"));
    text = reinterpret_cast<TextFn>(dlsym(lib, "sqlite3_column_text"));
    int64 = reinterpret_cast<Int64Fn>(dlsym(lib, "sqlite3_column_int64"));
    finalize = reinterpret_cast<FinalizeFn>(dlsym(lib, "sqlite3_finalize"));
    close = reinterpret_cast<CloseFn>(dlsym(lib, "sqlite3_close"));
    errmsg = reinterpret_cast<ErrFn>(dlsym(lib, "sqlite3_errmsg"));
    if (open && prepare && step && text && int64 && finalize && close && errmsg) return true;
    open = nullptr;
    return false;
  }
};
Sqlite g_sqlite;
constexpr int kSqliteOk = 0, kSqliteRow = 100, kSqliteDone = 101, kSqliteOpenReadonly = 1;

inline uint16_t rd16(const uint8_t* p) { uint16_t v; memcpy(&v, p, 2); return v; }
inline uint32_t rd32(const uint8_t* p) { uint32_t v; memcpy(&v, p, 4); return v; }
}  // namespace

BgenFile::~BgenFile() {
  if (data) munmap(const_cast<uint8_t*>(data), size);
  if (fd >= 0) close(fd);
}

void BgenFile::open(const std::string& p, const std::string& sample_file, bool ref_first,
                    const std::set<std::string>& exclude, const std::set<std::string>& extract,
                    const std::set<std::string>& remove, const std::set<std::string>& keep, const std::set<int>& chrs,
                    const std::string& bgi_file, bool no_bgi) {
  path = p;
  fd = ::open(path.c_str(), O_RDONLY);
  if (fd < 0) throw Fail("cannot open file : " + path);
  struct stat st;
  fstat(fd, &st);
  size = (size_t)st.st_size;
  if (size < 24) throw Fail("bgen file is too short : " + path);
  void* m = mmap(nullptr, size, PROT_READ, MAP_PRIVATE, fd, 0);
  if (m == MAP_FAILED) throw Fail("cannot map file : " + path);
  data = static_cast<const uint8_t*>(m);
  const uint32_t offset = rd32(data), lh = rd32(data + 4);
  n_variants_file = rd32(data + 8);
  n_file = rd32(data + 12);
  if (memcmp(data + 16, "bgen", 4) != 0 && memcmp(data + 16, "\0\0\0\0", 4) != 0) throw Fail("not a bgen file : " + path);
  if (lh < 20 || (uint64_t)4 + lh > size || (uint64_t)offset + 4 > size || offset < lh)
    throw Fail("corrupt bgen header (block lengths do not fit the file) : " + path);
  const uint32_t flags = rd32(data + 4 + lh - 4);
  compression = flags & 3;
  const int layout = (flags >> 2) & 0xF;
  const bool has_ids = (flags >> 31) != 0;
  if (layout != 2) throw Fail("only BGEN v1.2 (layout 2) files are supported.");
  if (compression > 2) throw Fail("unknown bgen compression flag.");
  if (compression == 2) load_zstd();
  // ---- sample identifiers: embedded block, or --sample (read_bgen_sample, src/Geno.cpp:391-440)
  if (!sample_file.empty()) {
    LineReader fh(sample_file);
    std::string line;
    int lineno = 0;
    while (fh.getline(line)) {
      auto t = split_ws(line);
      if (t.empty()) continue;
      if (lineno++ < 2) {
        if (lineno == 1 && (t.size() < 2 || t[0] != "ID_1" || t[1] != "ID_2")) throw Fail("header of the sample file must start with: ID_1 ID_2");
        continue;
      }
      if (t.size() < 2) throw Fail("incorrectly formatted sample file.");
      keys_file.push_back(t[0] + "_" + t[1]);
      ids_file.emplace_back(t[0], t[1]);
      sex_file.push_back(t.size() >= 4 ? (t[3] == "1" ? 1 : (t[3] == "2" ? 2 : 0)) : 0);   // src/Geno.cpp:395-456
    }
    if (keys_file.size() != n_file) throw Fail("number of samples in BGEN file does not match that in the sample file.");
  } else {
    if (!has_ids) throw Fail("the bgen file has no sample identifiers: provide them with --sample.");
    const uint8_t* q = data + 4 + lh;
    if ((uint64_t)4 + lh + 8 > (uint64_t)offset + 4) throw Fail("corrupt sample identifier block in bgen file.");
    const uint32_t ns = rd32(q + 4);
    if (ns != n_file) throw Fail("inconsistent sample identifier block in bgen file.");
    q += 8;
    const uint8_t* const qend = data + (size_t)offset + 4;   // the sample block ends where the variant blocks start
    for (uint32_t i = 0; i < ns; ++i) {
      if (q + 2 > qend) throw Fail("corrupt sample identifier block in bgen file.");
      const uint16_t l = rd16(q);
      if (q + 2 + l > qend) throw Fail("corrupt sample identifier block in bgen file.");
      keys_file.emplace_back(reinterpret_cast<const char*>(q + 2), l);
      sex_file.push_back(0);
      q += 2 + l;
    }
  }
  {
    std::set<std::string> seen;
    for (const auto& k : keys_file)
      if (!seen.insert(k).second) throw Fail("duplicate individual in bgen file : FID_IID =" + k);
  }
  for (size_t i = 0; i < keys_file.size(); ++i) {
    const std::string& k = keys_file[i];
    if (remove.count(k)) continue;
    if (!keep.empty() && !keep.count(k)) continue;
    if (sex_specific && sex_file[i] != sex_specific) continue;   // --sex-specific (src/Geno.cpp:1287-1293)
    key_to_ind[k] = (uint32_t)keys.size();
    keys.push_back(k);
    sample_idx.push_back((int32_t)i);
  }
  if (keys.empty()) throw Fail("no samples left after --keep/--remove/--sex-specific.");
  // ---- variant index: one variant identifying block at file position `pos` (BGEN v1.2 spec); leaves `pos` at the
  // genotype block and returns false when the variant is filtered out
  size_t pos = 0;
  auto need = [&](size_t n) { if (pos + n > size) throw Fail("unexpected end of bgen file."); };
  auto parse_variant = [&](Snp& s) {
    need(2); uint16_t l = rd16(data + pos); pos += 2 + l;                                 // SNPID
    need(2); l = rd16(data + pos); need(2 + l); s.id.assign(reinterpret_cast<const char*>(data + pos + 2), l); pos += 2 + l;
    need(2); l = rd16(data + pos); need(2 + l);
    const std::string chrom(reinterpret_cast<const char*>(data + pos + 2), l); pos += 2 + l;
    need(6); s.pos = rd32(data + pos); pos += 4;
    const uint16_t k = rd16(data + pos); pos += 2;
    if (k != 2) throw Fail("only bi-allelic variants are supported in bgen files (variant " + s.id + ").");
    std::string al[2];
    for (int a = 0; a < 2; ++a) {
      need(4); const uint32_t la = rd32(data + pos); need(4 + la);
      al[a].assign(reinterpret_cast<const char*>(data + pos + 4), la); pos += 4 + la;
    }
    s.chrom = chr_str_to_int(chrom);
    if (s.chrom == -1) throw Fail("unknown chromosome code in bgen file.");
    if (ref_first) { s.allele0 = al[0]; s.allele1 = al[1]; }
    else           { s.allele0 = al[1]; s.allele1 = al[0]; }    // allele0 of the file is ALT
    s.offset = pos;
    need(4); const uint32_t c = rd32(data + pos);
    need(4 + (size_t)c);
    pos += 4 + (size_t)c;
    if (!chrs.empty() && !chrs.count(s.chrom)) return false;
    if (exclude.count(s.id)) return false;
    if (!extract.empty() && !extract.count(s.id)) return false;
    return true;
  };
  // with an index file the variant start positions come from its Variant table (read_bgi_file, src/Geno.cpp:180-309);
  // the identifying block at each position is still parsed (an O(1) hop in the mapping) because the genotype block
  // offset is what read_block needs, and it doubles as the reference's consistency check of index against file
  std::string bgi = bgi_file.empty() ? path + ".bgi" : bgi_file;
  struct stat bst;
  const bool have_bgi = !no_bgi && stat(bgi.c_str(), &bst) == 0;
  if (!bgi_file.empty() && !have_bgi) throw Fail("cannot open file : " + bgi_file);
  if (have_bgi && g_sqlite.load()) {
    void *db = nullptr, *stmt = nullptr;
    if (g_sqlite.open(bgi.c_str(), &db, kSqliteOpenReadonly, nullptr) != kSqliteOk) {
      const std::string msg = db ? g_sqlite.errmsg(db) : "out of memory";
      if (db) g_sqlite.close(db);
      throw Fail("cannot open index file " + bgi + " (" + msg + ")");
    }
    if (g_sqlite.prepare(db, "SELECT rsid, file_start_position, size_in_bytes FROM Variant", -1, &stmt, nullptr) != kSqliteOk) {
      const std::string msg = g_sqlite.errmsg(db);
      g_sqlite.close(db);
      throw Fail("failed reading file (" + msg + ").");
    }
    std::vector<std::pair<uint64_t, uint64_t>> starts;                                   // (file position, size)
    std::vector<std::string> ids;
    int rc;
    while ((rc = g_sqlite.step(stmt)) == kSqliteRow) {
      const unsigned char* t = g_sqlite.text(stmt, 0);
      ids.emplace_back(t ? reinterpret_cast<const char*>(t) : "");
      starts.emplace_back((uint64_t)g_sqlite.int64(stmt, 1), (uint64_t)g_sqlite.int64(stmt, 2));
    }
    const std::string msg = rc == kSqliteDone ? "" : g_sqlite.errmsg(db);
    g_sqlite.finalize(stmt);
    g_sqlite.close(db);
    if (rc != kSqliteDone) throw Fail("failed reading file (" + msg + ").");
    if (starts.size() != n_variants_file) throw Fail("the bgi index does not match the bgen file (number of variants).");
    // the Variant table is keyed by (chromosome TEXT, position, ...): rows come back in that order, which is the file
    // order whenever chromosome names sort like their numbers; blocks need file order, so restore it in any case
    std::vector<size_t> order(starts.size());
    for (size_t i = 0; i < order.size(); ++i) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](size_t a, size_t b) { return starts[a].first < starts[b].first; });
    for (size_t i : order) {
      Snp s;
      pos = (size_t)starts[i].first;
      if (pos < (size_t)offset + 4) throw Fail("the bgi index does not match the bgen file (variant position).");
      const bool keep_it = parse_variant(s);
      if (s.id != ids[i] || pos - (size_t)starts[i].first != (size_t)starts[i].second)
        throw Fail("the bgi index does not match the bgen file (variant " + ids[i] + ").");
      if (keep_it) snps.push_back(s);
    }
    used_bgi = true;
    return;
  }
  pos = (size_t)offset + 4;
  for (uint32_t v = 0; v < n_variants_file; ++v) {
    Snp s;
    if (parse_variant(s)) snps.push_back(s);
  }
}

void BgenFile::read_block(size_t first, size_t n, uint8_t* probs, uint8_t* pm, int threads) const {
  std::atomic<size_t> next{0};
  std::string err;
  std::atomic<bool> failed{false};
  auto work = [&]() {
    std::vector<uint8_t> buf;
    for (;;) {
      const size_t j = next.fetch_add(1);
      if (j >= n || failed.load()) return;
      const uint8_t* q = data + snps[first + j].offset;
      const uint32_t c = rd32(q);
      const uint8_t* raw;
      uLongf dl;
      const size_t want = 10 + 3 * (size_t)n_file;          // the only payload this reader accepts (8-bit, ploidy 2, biallelic)
      // lengths come from the file: validate them BEFORE they size a buffer or a source span (same rules as
      // read_block_compressed); parse_variant already checked that the c bytes lie inside the mapping
      if (compression != 0) {
        if (c < 8) { failed = true; return; }
        dl = rd32(q + 4);
        if ((size_t)dl != want) { failed = true; return; }
        buf.resize(dl);
      }
      if (compression == 1) {
        if (uncompress(buf.data(), &dl, q + 8, c - 4) != Z_OK || (size_t)dl != want) { failed = true; return; }
        raw = buf.data();
      } else if (compression == 2) {
        const size_t got = g_zstd_decompress(buf.data(), dl, q + 8, c - 4);
        if (g_zstd_is_error(got) || got != want) { failed = true; return; }
        raw = buf.data();
      } else {
        dl = c;
        if ((size_t)dl != want) { failed = true; return; }
        raw = q + 4;
      }
      const uint32_t ns = rd32(raw);
      const uint16_t ka = rd16(raw + 4);
      const uint8_t pmin = raw[6], pmax = raw[7];
      if (ns != n_file || ka != 2 || pmin != 2 || pmax != 2) { failed = true; return; }
      const uint8_t phased = raw[8 + ns], bits = raw[9 + ns];
      if (phased != 0 || bits != 8) { failed = true; return; }
      memcpy(pm + j * (size_t)n_file, raw + 8, ns);
      memcpy(probs + j * (size_t)n_file * 2, raw + 10 + ns, 2 * (size_t)ns);
    }
  };
  const int T = (int)std::max<size_t>(1, std::min<size_t>((size_t)threads, n));
  std::vector<std::thread> pool;
  for (int t = 1; t < T; ++t) pool.emplace_back(work);
  work();
  for (auto& t : pool) t.join();
  if (failed) throw Fail("unsupported or corrupt bgen genotype block (rgb200 reads 8-bit unphased diploid biallelic layout 2 only).");
}

void BgenFile::info_all(const uint8_t* probs, const uint8_t* pm, size_t n, const uint8_t* in_analysis, bool ref_first,
                        double* info_out, int threads) const {
  std::atomic<size_t> next{0};
  const size_t nk = sample_idx.size();
  auto work = [&]() {
    for (;;) {
      const size_t j = next.fetch_add(1);
      if (j >= n) return;
      const uint8_t* pr = probs + j * (size_t)n_file * 2;
      const uint8_t* m = pm + j * (size_t)n_file;
      // integer sums in units of 1/255 (dosage) and 1/255^2 (its square): exact, order-independent
      uint64_t s_d = 0, s_d2 = 0, s_e = 0, ns = 0;
      for (size_t k = 0; k < nk; ++k) {
        if (!in_analysis[k]) continue;
        const size_t f = (size_t)sample_idx[k];
        if (m[f] & 0x80) continue;
        const uint32_t p0 = pr[2 * f], p1 = pr[2 * f + 1];
        const uint32_t hom = ref_first ? (p0 + p1 > 255 ? 0 : 255 - p0 - p1) : p0;
        const uint32_t d = p1 + 2 * hom;
        s_d += d;
        s_d2 += (uint64_t)d * d;
        s_e += 4 * hom + p1;
        ++ns;
      }
      if (ns == 0) { info_out[j] = 1.0; continue; }
      const double total = (double)s_d / 255.0, af = total / (2.0 * (double)ns);
      const double info_num = (double)s_e / 255.0 - (double)s_d2 / 65025.0;
      info_out[j] = (af == 0.0 || af == 1.0) ? 1.0 : 1.0 - info_num / (2.0 * (double)ns * af * (1.0 - af));
    }
  };
  const int T = (int)std::max<size_t>(1, std::min<size_t>((size_t)threads, n));
  std::vector<std::thread> pool;
  for (int t = 1; t < T; ++t) pool.emplace_back(work);
  work();
  for (auto& t : pool) t.join();
}

void BgenFile::read_block_compressed(size_t first, size_t n, std::vector<uint8_t>& comp, std::vector<uint64_t>& offs) const {
  if (compression != 1) throw Fail("on-device inflate needs zlib-compressed bgen payloads (compression flag 1).");
  offs.assign(n + 1, 0);
  size_t total = 0;
  for (size_t j = 0; j < n; ++j) {
    const uint8_t* q = data + snps[first + j].offset;
    const uint32_t c = rd32(q), d = rd32(q + 4);
    if (c < 4 || (uint64_t)d != 10 + 3 * (uint64_t)n_file)
      throw Fail("unsupported or corrupt bgen genotype block (rgb200 reads 8-bit unphased diploid biallelic layout 2 only).");
    total += c - 4;
    offs[j + 1] = total;
  }
  comp.resize(total);
  for (size_t j = 0; j < n; ++j) {
    const uint8_t* q = data + snps[first + j].offset;
    memcpy(comp.data() + offs[j], q + 8, (size_t)(offs[j + 1] - offs[j]));
  }
}

}  // namespace rgh
