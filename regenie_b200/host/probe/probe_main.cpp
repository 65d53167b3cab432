// rgb200_hostprobe -- test hook for the host-side logic of the rgb200 driver (readers, phenotype preparation, null
// models, text formats).  It links the same translation units as the driver (everything under host/ except main.cpp),
// never touches the GPU library, and prints / dumps what those functions produce so that the CPU test suite
// (tests/test_host_cpu.py) can compare them with the oracle without a CUDA device.  Not part of the product path.
//
//   rgb200_hostprobe bgen-variants FILE [--bgi F] [--no-bgi] [--ref-first] [--sample F] [--chr C]...
//   rgb200_hostprobe bgen-probs FILE FIRST N OUT            raw probability + ploidy bytes of N variants
//   rgb200_hostprobe bgen-info FILE [--ref-first]           variant-level INFO (info1) of every variant
//   rgb200_hostprobe rows (--bed|--pgen) PREFIX OUT          every variant as PLINK 1 2-bit rows
//   rgb200_hostprobe counts CLASSES OUT (--bed PREFIX|--bgen FILE) [--ref-first] [--remove F]
//                    genotype counts of every variant (host/counts.hpp), int64 [variants][T][6].  CLASSES: a line
//                    "T binary male non_par", then cls [T][kept samples], male [kept samples] if male = 1 and
//                    non_par [variants] if non_par = 1, one byte each
//   rgb200_hostprobe prep OUT (--bed|--pgen|--bgen) X --phenoFile F [--covarFile F] [--bt] [--step2] [--strict]
//                    [--remove F] [--keep F] [--apply-rint] [--catCovarList a,b] [--phenoColList a,b] [--covarColList a,b]
//                    [--cv K] [--bsize B] [--null-eta]
//   rgb200_hostprobe cat FILE                               lines through LineReader (plain or .gz)
//   rgb200_hostprobe pred-file OUT N [--prs]                a prediction file of deterministic values (N samples)
//   rgb200_hostprobe read-pred FILE [--prs]                 ids + rows back out, one token per line
//   rgb200_hostprobe sumstats                               stdin: "af info n beta se chisq pass" per line -> rows
//   rgb200_hostprobe ids OUT NAME PRINTNAME                 stdin: "FID IID keep" per line
//   rgb200_hostprobe inflate-bgen FILE [window]             every zlib payload through csrc/inflate_core.h vs zlib
//   rgb200_hostprobe inflate IN OUTLEN OUT [window]         one zlib stream through csrc/inflate_core.h (status on stdout)
//                                                           `window` selects inflate_zlib_window (ring in shared memory)
#include <cstring>
#include <iomanip>

#include <zlib.h>

#include "../../csrc/inflate_core.h"
#include "../../csrc/pgen_core.h"
#include "../bgen.hpp"
#include "../bt_null.hpp"
#include "../counts.hpp"
#include "../data.hpp"
#include "../output.hpp"
#include "../pgen.hpp"

using namespace rgh;

namespace {

std::set<std::string> csv_set(const std::string& v) {
  std::set<std::string> out;
  std::string tok;
  std::istringstream ss(v);
  while (std::getline(ss, tok, ',')) if (!tok.empty()) out.insert(tok);
  return out;
}

template <typename T>
void dump(std::ofstream& f, const char* name, const std::vector<T>& v, const char* dtype) {
  f << name << " " << dtype << " " << v.size() << "\n";
  f.write(reinterpret_cast<const char*>(v.data()), (std::streamsize)(v.size() * sizeof(T)));
  f << "\n";
}

int cmd_bgen_variants(int argc, char** argv) {
  std::string bgi, sample;
  bool no_bgi = false, ref_first = false;
  std::set<int> chrs;
  for (int i = 3; i < argc; ++i) {
    const std::string a = argv[i];
    if (a == "--bgi") bgi = argv[++i];
    else if (a == "--no-bgi") no_bgi = true;
    else if (a == "--ref-first") ref_first = true;
    else if (a == "--sample") sample = argv[++i];
    else if (a == "--chr") chrs.insert(chr_str_to_int(argv[++i]));
  }
  BgenFile g;
  g.open(argv[2], sample, ref_first, {}, {}, {}, {}, chrs, bgi, no_bgi);
  std::cout << "used_bgi " << g.used_bgi << " n_file " << g.n_file << " compression " << g.compression << "\n";
  for (const auto& s : g.snps)
    std::cout << s.chrom << " " << s.id << " " << s.pos << " " << s.allele0 << " " << s.allele1 << " " << s.offset << "\n";
  return 0;
}

int cmd_bgen_probs(char** argv) {
  BgenFile g;
  g.open(argv[2], "", false, {}, {}, {}, {}, {}, "", true);
  const size_t first = (size_t)atol(argv[3]), n = (size_t)atol(argv[4]);
  std::vector<uint8_t> probs(n * g.n_file * 2), pm(n * g.n_file);
  g.read_block(first, n, probs.data(), pm.data(), 4);
  std::ofstream f(argv[5], std::ios::binary);
  f.write(reinterpret_cast<const char*>(probs.data()), (std::streamsize)probs.size());
  f.write(reinterpret_cast<const char*>(pm.data()), (std::streamsize)pm.size());
  return 0;
}

// variant-level INFO of every variant (all samples analysed), one value per line
int cmd_bgen_info(int argc, char** argv) {
  const bool ref_first = argc > 3 && std::string(argv[3]) == "--ref-first";
  BgenFile g;
  g.open(argv[2], "", ref_first, {}, {}, {}, {}, {}, "", true);
  const size_t n = g.snps.size();
  std::vector<uint8_t> probs(n * g.n_file * 2), pm(n * g.n_file), ina(g.keys.size(), 1);
  g.read_block(0, n, probs.data(), pm.data(), 4);
  std::vector<double> info(n);
  g.info_all(probs.data(), pm.data(), n, ina.data(), ref_first, info.data(), 4);
  std::cout << std::setprecision(17);
  for (double v : info) std::cout << v << "\n";
  return 0;
}

int cmd_rows(char** argv) {
  BedFile g;
  if (std::string(argv[2]) == "--pgen") g.open_pgen(argv[3], {}, {}, {}, {}, {});
  else g.open(argv[3], false, {}, {}, {}, {}, {});
  std::vector<uint8_t> rows(g.snps.size() * g.row_stride);
  g.read_rows(0, g.snps.size(), rows.data());
  std::ofstream f(argv[4], std::ios::binary);
  f.write(reinterpret_cast<const char*>(rows.data()), (std::streamsize)rows.size());
  std::cout << g.snps.size() << " " << g.row_stride << " " << g.keys.size() << "\n";
  return 0;
}

// the hard-call counter on the rows of a .bed, or the dosage counter on the probability pairs of a .bgen
int cmd_counts(int argc, char** argv) {
  std::string bed, bgen, remove;
  bool ref_first = false;
  for (int i = 4; i < argc; ++i) {
    const std::string a = argv[i];
    if (a == "--bed") bed = argv[++i];
    else if (a == "--bgen") bgen = argv[++i];
    else if (a == "--remove") remove = argv[++i];
    else if (a == "--ref-first") ref_first = true;
    else throw Fail("probe: unknown option " + a);
  }
  BedFile g;
  BgenFile gg;
  const auto rem = read_id_list(remove, 2);
  if (!bgen.empty()) gg.open(bgen, "", ref_first, {}, {}, rem, {}, {}, "", true);
  else g.open(bed, ref_first, {}, {}, rem, {});
  const std::vector<int32_t>& sidx = bgen.empty() ? g.sample_idx : gg.sample_idx;
  const size_t M = bgen.empty() ? g.snps.size() : gg.snps.size(), N = sidx.size();
  const size_t n_file = bgen.empty() ? g.keys_file.size() : gg.n_file;
  ClassTable ct;
  int binary = 0, has_male = 0, has_np = 0;
  std::ifstream f(argv[2], std::ios::binary);
  f >> ct.T >> binary >> has_male >> has_np;
  f.get();
  ct.binary = binary != 0;
  auto bytes = [&](std::vector<uint8_t>& v, size_t n) {
    v.resize(n);
    f.read(reinterpret_cast<char*>(v.data()), (std::streamsize)n);
  };
  std::vector<uint8_t> non_par;
  bytes(ct.cls, (size_t)ct.T * N);
  if (has_male) bytes(ct.male, N);
  if (has_np) bytes(non_par, M);
  if (!f) throw Fail("probe: class file too short");
  const uint8_t* np = has_np ? non_par.data() : nullptr;
  std::vector<long> out(M * ct.T * 6);
  if (!bgen.empty()) {
    std::vector<uint8_t> probs(M * n_file * 2), pm(M * n_file);
    gg.read_block(0, M, probs.data(), pm.data(), 4);
    dosage_counts(ct, ref_first, n_file, sidx, probs.data(), pm.data(), M, np, out.data(), 4);
  } else {
    std::vector<uint8_t> rows(M * g.row_stride);
    g.read_rows(0, M, rows.data());
    HardCallCounts hc;
    hc.init(ct, ref_first, n_file, sidx);
    hc.count(rows.data(), g.row_stride, (int)M, np, out.data(), 4);
  }
  std::ofstream o(argv[3], std::ios::binary);
  for (long x : out) {
    const int64_t v = x;
    o.write(reinterpret_cast<const char*>(&v), sizeof(v));
  }
  std::cout << M << " " << N << " " << n_file << "\n";
  return 0;
}

// The device decoder's arithmetic (csrc/pgen_core.h) on the host, lanes of a warp one after the other, fed exactly like
// rg_pgen_decode: PgenFile::gather per block of `bs` variants, rows written with the .bed stride for comparison with `rows`.
int cmd_pgen_rows(char** argv) {
  BedFile g;
  g.open_pgen(argv[2], {}, {}, {}, {}, {});
  const size_t bs = (size_t)atoi(argv[4]), m = g.snps.size();
  const uint32_t n = g.pg->n_file, words = ((n + 15) / 16 + 3) / 4 * 4;
  std::vector<uint8_t> rows(m * g.row_stride);
  std::vector<uint32_t> row(words);
  PgenBatch pb;
  size_t nrec = 0, nbytes = 0;
  for (size_t first = 0; first < m; first += bs) {
    const size_t cnt = std::min(bs, m - first);
    g.pg->gather(first, cnt, pb);
    nrec += pb.rec_off.size(); nbytes += pb.bytes.size();
    for (size_t j = 0; j < cnt; ++j) {
      auto rec = [&](int32_t r) { return rgp::Rec{pb.bytes.data() + pb.rec_off[r], pb.rec_len[r], pb.rec_type[r]}; };
      const rgp::Rec own = rec(pb.own[j]);
      rgp::Rec base{nullptr, 0, 0};
      if (pb.base[j] >= 0) base = rec(pb.base[j]);
      const int e = rgp::decode_row_serial(own, pb.base[j] >= 0 ? &base : nullptr, n, row.data(), words, 32);
      if (e) throw Fail("pgen core: error " + std::to_string(e) + " at variant " + std::to_string(first + j));
      memcpy(&rows[(first + j) * g.row_stride], row.data(), g.row_stride);
    }
  }
  std::ofstream f(argv[3], std::ios::binary);
  f.write(reinterpret_cast<const char*>(rows.data()), (std::streamsize)rows.size());
  std::cout << m << " " << g.row_stride << " " << g.keys.size() << " " << nrec << " " << nbytes << "\n";
  return 0;
}

int cmd_prep(int argc, char** argv) {
  std::string bed, pgen, bgen, pheno, covar, remove, keep;
  bool bt = false, step2 = false, strict = false, null_eta = false;
  int cv = 5, bsize = 100;
  Pheno ph;
  for (int i = 3; i < argc; ++i) {
    const std::string a = argv[i];
    if (a == "--bed") bed = argv[++i];
    else if (a == "--pgen") pgen = argv[++i];
    else if (a == "--bgen") bgen = argv[++i];
    else if (a == "--phenoFile") pheno = argv[++i];
    else if (a == "--covarFile") covar = argv[++i];
    else if (a == "--remove") remove = argv[++i];
    else if (a == "--keep") keep = argv[++i];
    else if (a == "--bt") bt = true;
    else if (a == "--step2") step2 = true;
    else if (a == "--strict") strict = true;
    else if (a == "--apply-rint") ph.rint = true;
    else if (a == "--catCovarList") ph.cat_cols = csv_set(argv[++i]);
    else if (a == "--phenoColList") ph.pheno_cols = csv_set(argv[++i]);
    else if (a == "--covarColList") ph.covar_cols = csv_set(argv[++i]);
    else if (a == "--cv") cv = atoi(argv[++i]);
    else if (a == "--bsize") bsize = atoi(argv[++i]);
    else if (a == "--null-eta") null_eta = true;
    else throw Fail("probe: unknown option " + a);
  }
  BedFile g;
  BgenFile gg;
  const auto rem = read_id_list(remove, 2), kp = read_id_list(keep, 2);
  if (!bgen.empty()) gg.open(bgen, "", false, {}, {}, rem, kp);
  else if (!pgen.empty()) g.open_pgen(pgen, {}, {}, rem, kp);
  else g.open(bed, false, {}, {}, rem, kp);
  const std::vector<std::string>& keys = bgen.empty() ? g.keys : gg.keys;
  const std::vector<Snp>& snps = bgen.empty() ? g.snps : gg.snps;
  Log log;
  read_pheno_and_cov(SampleSet{keys, bgen.empty() ? g.key_to_ind : gg.key_to_ind}, pheno, covar, step2, strict, bt, ph, log);
  prep_run(ph, nullptr, log);
  std::ofstream f(argv[2], std::ios::binary);
  f << "N " << ph.N << " P " << ph.P << " C " << ph.C << " n_analyzed " << ph.n_analyzed << " strict " << ph.strict << "\n";
  f << "names";
  for (auto& n : ph.names) f << " " << n;
  f << "\n";
  dump(f, "X", ph.X, "f8");
  dump(f, "Y", ph.Y, "f8");
  dump(f, "Y_raw", ph.Y_raw, "f8");
  dump(f, "mask", ph.mask, "u1");
  dump(f, "in_analysis", ph.in_analysis, "u1");
  dump(f, "neff", ph.neff, "f8");
  dump(f, "scale_Y", ph.scale_Y, "f8");
  dump(f, "folds", set_folds(ph.in_analysis, cv), "i8");
  std::vector<int64_t> blk;
  for (const auto& b : set_blocks(snps, bsize)) { blk.push_back(b.chrom); blk.push_back((int64_t)b.first); blk.push_back(b.size); }
  dump(f, "blocks", blk, "i8");
  if (null_eta && bt) {
    std::vector<double> eta;
    for (int i = 0; i < ph.P; ++i) {
      const auto e = null_logistic_eta(ph.names[i], &ph.Y_raw[(size_t)i * ph.N], ph.X.data(), ph.N, ph.C, &ph.mask[(size_t)i * ph.N]);
      eta.insert(eta.end(), e.begin(), e.end());
    }
    dump(f, "null_eta", eta, "f8");
  }
  return 0;
}

int cmd_cat(char** argv) {
  LineReader r(argv[2]);
  std::string line;
  while (r.getline(line)) std::cout << line << "\n";
  return 0;
}

int cmd_pred_file(int argc, char** argv) {
  const int n = atoi(argv[3]);
  const bool prs = argc > 4 && std::string(argv[4]) == "--prs";
  std::vector<std::string> keys(n);
  std::vector<uint32_t> order;
  std::vector<uint8_t> mask(n);
  for (int i = 0; i < n; ++i) { keys[i] = "F" + std::to_string(i) + "_I" + std::to_string(i); mask[i] = (i % 7) != 3; }
  std::map<std::string, uint32_t> m;
  for (int i = 0; i < n; ++i) if (i % 11 != 5) m[keys[i]] = (uint32_t)i;       // "analysed" samples in std::map key order
  for (auto& kv : m) order.push_back(kv.second);
  const int R = prs ? 1 : 23;
  std::vector<double> vals((size_t)R * n);
  for (int r = 0; r < R; ++r)
    for (int i = 0; i < n; ++i) vals[(size_t)r * n + i] = std::sin(0.37 * (r + 1) * (i + 1)) * std::pow(10.0, (i % 13) - 6);
  std::vector<int> labels;
  std::vector<const double*> rows;
  for (int r = 0; r < R; ++r) { labels.push_back(prs ? 0 : r + 1); rows.push_back(&vals[(size_t)r * n]); }
  TextWriter w;
  w.open(argv[2]);
  write_pred_file(w, keys, order, mask.data(), labels, rows);
  w.close();
  return 0;
}

int cmd_read_pred(int argc, char** argv) {
  const bool prs = argc > 3 && std::string(argv[3]) == "--prs";
  Loco l = read_loco(argv[2], prs);
  std::cout << "ids " << l.ids.size() << "\n";
  for (auto& s : l.ids) std::cout << s << "\n";
  auto show = [](double v) { if (std::isnan(v)) std::cout << "NA\n"; else std::cout << v << "\n"; };
  std::cout << "first " << l.first.size() << "\n";
  for (double v : l.first) show(v);
  // rows on demand, out of file order on purpose (a plain file seeks, a .gz file was parsed when it was opened)
  for (int c = 23; c >= 1; --c) {
    if (!l.has_row(c)) continue;
    const std::vector<double>& r = l.row(c);
    std::cout << "row " << c << " " << r.size() << "\n";
    for (double v : r) show(v);
    if (prs) break;
  }
  return 0;
}

int cmd_sumstats() {
  std::string line;
  std::cout << sumstats_header(true) << sumstats_header(false);
  while (std::getline(std::cin, line)) {
    auto t = split_ws(line);
    if (t.size() != 7) continue;
    const double af = atof(t[0].c_str()), info = atof(t[1].c_str()), beta = atof(t[3].c_str()), se = atof(t[4].c_str()),
                 chisq = atof(t[5].c_str());
    const int n = atoi(t[2].c_str());
    const bool pass = t[6] == "1";
    std::cout << sumstats_row("1 100 rs1 A G ", af, true, info, n, "ADD", beta, se, chisq, get_logp(chisq), pass);
    std::cout << sumstats_row("23 5 rs2 AT G ", af, false, -1.0, n, "ADD", beta, se, chisq, get_logp(chisq), pass);
    std::cout << std::setprecision(17) << get_logp(chisq) << "\n" << std::setprecision(6);
  }
  return 0;
}

// stdin lines: bt firth pass beta se chisq logp af mac gc0..gc5 score skat_var cal_factor info  (info < 0: none) -> HTP rows
int cmd_htp() {
  std::string line;
  std::cout << htp_header();
  while (std::getline(std::cin, line)) {
    auto t = split_ws(line);
    if (t.size() != 19) continue;
    HtpRow r;
    r.bt = t[0] == "1"; r.firth = t[1] == "1"; r.test_pass = t[2] == "1";
    r.beta = strtod(t[3].c_str(), nullptr); r.se = strtod(t[4].c_str(), nullptr); r.chisq = strtod(t[5].c_str(), nullptr);
    r.logp = strtod(t[6].c_str(), nullptr); r.af = strtod(t[7].c_str(), nullptr); r.mac = strtod(t[8].c_str(), nullptr);
    for (int k = 0; k < 6; ++k) r.gc[k] = atol(t[9 + k].c_str());
    r.score = strtod(t[15].c_str(), nullptr); r.skat_var = strtod(t[16].c_str(), nullptr); r.cal_factor = strtod(t[17].c_str(), nullptr);
    r.info = strtod(t[18].c_str(), nullptr);
    r.model = r.bt ? (r.firth ? "ADD-WGR-FIRTH" : "ADD-WGR-LOG") : "ADD-WGR-LR";
    std::string out;
    append_htp_row(out, "rs1\t1\t100\tA\tG\t", "Y1", "COHORT", r);
    std::cout << out;
  }
  return 0;
}

int cmd_ids(char** argv) {
  std::vector<std::pair<std::string, std::string>> ids;
  std::vector<uint8_t> mask;
  std::string line;
  while (std::getline(std::cin, line)) {
    auto t = split_ws(line);
    if (t.size() != 3) continue;
    ids.emplace_back(t[0], t[1]);
    mask.push_back(t[2] == "1");
  }
  write_ids_file(argv[2], argv[3], std::string(argv[4]) == "1", ids, mask.data());
  return 0;
}

// the decoder the GPU runs (csrc/inflate_core.h, compiled here with a one-lane "warp") against zlib on every variant
// one stream through the selected variant of the decoder
int run_inflate(bool window, const uint8_t* in, uint32_t n, uint8_t* out, uint32_t out_len) {
  static rgi::Tables t;
  static std::vector<uint8_t> win(rgi::kWinBytes);
  return window ? rgi::inflate_zlib_window(in, n, out, out_len, t, win.data(), true) : rgi::inflate_zlib(in, n, out, out_len, t, true);
}

int cmd_inflate_bgen(int argc, char** argv) {
  const bool window = argc > 3 && std::string(argv[3]) == "window";
  BgenFile g;
  g.open(argv[2], "", false, {}, {}, {}, {}, {}, "", true);
  std::vector<uint8_t> comp;
  std::vector<uint64_t> offs;
  g.read_block_compressed(0, g.snps.size(), comp, offs);
  const uint32_t raw_len = 10 + 3 * g.n_file;
  std::vector<uint8_t> a(raw_len), b(raw_len);
  size_t bad = 0, in_bytes = 0;
  for (size_t v = 0; v < g.snps.size(); ++v) {
    const uint32_t n = (uint32_t)(offs[v + 1] - offs[v]);
    in_bytes += n;
    std::fill(a.begin(), a.end(), 0xAA);
    const int st = run_inflate(window, comp.data() + offs[v], n, a.data(), raw_len);
    uLongf dl = raw_len;
    const int zr = uncompress(b.data(), &dl, comp.data() + offs[v], n);
    if (st != 0 || zr != Z_OK || dl != raw_len || a != b) {
      ++bad;
      std::cout << "variant " << v << " status " << st << " zlib " << zr << "\n";
    }
    // a truncated and a corrupted copy must be rejected, never crash
    if (v % 97 == 0 && n > 16) {
      std::vector<uint8_t> c(comp.begin() + (long)offs[v], comp.begin() + (long)offs[v + 1]);
      const int st_trunc = run_inflate(window, c.data(), n / 2, a.data(), raw_len);
      c[n / 2] ^= 0x5a;
      const int st_flip = run_inflate(window, c.data(), n, a.data(), raw_len);
      if (st_trunc == 0 || st_flip == 0) { ++bad; std::cout << "variant " << v << " damaged stream accepted\n"; }
    }
  }
  std::cout << "variants " << g.snps.size() << " bad " << bad << " compressed " << in_bytes << " raw " << (size_t)raw_len * g.snps.size() << "\n";
  return bad ? 1 : 0;
}

int cmd_inflate(int argc, char** argv) {
  const bool window = argc > 5 && std::string(argv[5]) == "window";
  std::ifstream f(argv[2], std::ios::binary | std::ios::ate);
  if (!f) throw Fail(std::string("cannot open file : ") + argv[2]);
  std::vector<uint8_t> in((size_t)f.tellg());
  f.seekg(0);
  f.read(reinterpret_cast<char*>(in.data()), (std::streamsize)in.size());
  const uint32_t out_len = (uint32_t)atol(argv[3]);
  std::vector<uint8_t> out(out_len);
  const int st = run_inflate(window, in.data(), (uint32_t)in.size(), out.data(), out_len);
  std::ofstream o(argv[4], std::ios::binary);
  o.write(reinterpret_cast<const char*>(out.data()), (std::streamsize)out.size());
  std::cout << "status " << st << "\n";
  return 0;
}

}  // namespace

int main(int argc, char** argv) {
  try {
    if (argc < 2) throw Fail("usage: rgb200_hostprobe <command> ...");
    const std::string c = argv[1];
    if (c == "bgen-variants" && argc >= 3) return cmd_bgen_variants(argc, argv);
    if (c == "bgen-probs" && argc == 6) return cmd_bgen_probs(argv);
    if (c == "bgen-info" && argc >= 3) return cmd_bgen_info(argc, argv);
    if (c == "rows" && argc == 5) return cmd_rows(argv);
    if (c == "pgen-rows" && argc == 5) return cmd_pgen_rows(argv);
    if (c == "counts" && argc >= 6) return cmd_counts(argc, argv);
    if (c == "prep" && argc >= 3) return cmd_prep(argc, argv);
    if (c == "cat" && argc == 3) return cmd_cat(argv);
    if (c == "pred-file" && argc >= 4) return cmd_pred_file(argc, argv);
    if (c == "read-pred" && argc >= 3) return cmd_read_pred(argc, argv);
    if (c == "sumstats") return cmd_sumstats();
    if (c == "htp") return cmd_htp();
    if (c == "ids" && argc == 5) return cmd_ids(argv);
    if (c == "inflate-bgen" && argc >= 3) return cmd_inflate_bgen(argc, argv);
    if (c == "inflate" && argc >= 5) return cmd_inflate(argc, argv);
    throw Fail("unknown probe command or wrong number of arguments: " + c);
  } catch (const std::exception& e) {
    std::cout << "ERROR: " << e.what() << "\n";
    return 1;
  }
}
