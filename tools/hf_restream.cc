// tools/hf_restream — rewrites the HF passes of an existing VarDCT file with LZ77 codes, or in one of synth_enc's
// entropy-code forms (--code), keeping everything else.
//
//   hf_restream IN.jxl OUT.jxl rle|match|prefix|ans-forms|configs
//
// The container boxes (jbrd included), the image and frame headers, LfGlobal, the LF groups, HfGlobal's dequant
// matrices and coefficient orders, and each pass group's HF preset and coefficient values stay bit for bit. Only the HF
// pass codes in HfGlobal (same context-to-cluster map, new histograms, LZ77 enabled), the HF bits of the pass-group
// sections and the TOC change. The values and their clusters come from one decode by the project's CPU oracle, traced
// through EntropyReader (JXLB_ENTROPY_TRACE in host/entropy.h); the new streams are written by synth_enc's LZ77 parser
// and ANS writer (lz77_parse, EntropyEncoder). The number of values the decoder takes from copies goes to stderr.
// The form modes keep the context-to-cluster map too (the traced values carry their cluster, not their context) and
// write the codes and streams in that form without LZ77; the writer's "code-form:" report goes to stderr.
//
// Not part of the product: test infrastructure (built with oracle/'s sources, see tools/hf_restream.py).
#define SYNTH_ENC_NO_MAIN
#include "synth_enc.cc"

#include <map>

#include "../jxl_oxide_b200/csrc/host/planner.h"

extern "C" void* jxlo_decode(const uint8_t* data, size_t size, int output_colour, int threads, int capture, int* status,
                             char* err, size_t err_cap);
extern "C" void jxlo_free(void* h);

namespace jxlb {
namespace {
struct TracedStream {
  size_t begin = 0, end = 0;  // bit positions: before the ANS state, after the last value
  std::vector<std::pair<uint32_t, uint32_t>> values;  // (cluster, value)
};
struct TracedCode {
  size_t begin = 0, end = 0;
  std::vector<uint8_t> cluster_map;
  uint32_t num_clusters = 0;
  bool lz77 = false;
};
const void* g_reader = nullptr;
std::map<size_t, TracedStream> g_streams;  // by begin position
TracedStream* g_cur = nullptr;
std::map<uint32_t, TracedCode> g_codes;     // by pass
}  // namespace

void entropy_trace_begin(const void* reader, size_t pos_bits) {
  g_reader = reader;
  g_cur = &g_streams[pos_bits];
  *g_cur = TracedStream();
  g_cur->begin = g_cur->end = pos_bits;
}
void entropy_trace_value(const void* reader, uint32_t cluster, uint32_t value, size_t pos_bits) {
  if (reader != g_reader || !g_cur) return;
  g_cur->values.push_back({cluster, value});
  g_cur->end = pos_bits;
}
void entropy_trace_hf_code(uint32_t pass, size_t begin_bits, size_t end_bits, const EntropyCode& code) {
  TracedCode& t = g_codes[pass];
  t.begin = begin_bits, t.end = end_bits, t.cluster_map = code.cluster_map, t.num_clusters = code.num_clusters;
  t.lz77 = code.lz77_enabled;
}
}  // namespace jxlb

namespace {
[[noreturn]] void die(const char* msg) {
  fprintf(stderr, "hf_restream: %s\n", msg);
  exit(1);
}

uint32_t be32(const uint8_t* p) { return uint32_t(p[0]) << 24 | uint32_t(p[1]) << 16 | uint32_t(p[2]) << 8 | p[3]; }

// bits [from, to) of `src` appended to `w`
void copy_bits(BitWriter& w, const std::vector<uint8_t>& src, size_t from, size_t to) {
  BitReader br(src.data(), src.size(), from);
  for (size_t n = to - from; n;) {
    const uint32_t k = uint32_t(std::min<size_t>(n, 32));
    w.write(int(k), br.read(k));
    n -= k;
  }
}
}  // namespace

int main(int argc, char** argv) {
  if (argc != 4) die("usage: hf_restream IN OUT rle|match|prefix|ans-forms|configs");
  HfLz77 opt;
  opt.mode = argv[3];
  const bool form = opt.mode == "prefix" || opt.mode == "ans-forms" || opt.mode == "configs";
  if (opt.mode != "rle" && opt.mode != "match" && !form) die("mode is rle, match, prefix, ans-forms or configs");
  if (form) g_code = opt.mode, atexit([] { g_report.print(); });
  std::vector<uint8_t> file;
  {
    FILE* f = fopen(argv[1], "rb");
    if (!f) die("cannot open the input");
    uint8_t buf[65536];
    for (size_t n; (n = fread(buf, 1, sizeof buf, f)) > 0;) file.insert(file.end(), buf, buf + n);
    fclose(f);
  }
  // ---- container: the codestream is the jxlc box or the jxlp boxes' payloads; a bare codestream is its own ----
  struct Box {
    size_t at, size, payload;  // payload: where the codestream bytes start (jxlp: after the index)
    bool codestream;
  };
  std::vector<Box> boxes;
  std::vector<uint8_t> cs;
  const bool bare = file.size() >= 2 && file[0] == 0xff && file[1] == 0x0a;
  if (bare) {
    cs = file;
  } else {
    for (size_t at = 0; at < file.size();) {
      if (at + 8 > file.size()) die("truncated box");
      size_t size = be32(&file[at]), head = 8;
      if (size == 1) die("64-bit box sizes are not written back");
      if (size == 0) size = file.size() - at;
      const std::string type(reinterpret_cast<const char*>(&file[at + 4]), 4);
      const bool is_cs = type == "jxlc" || type == "jxlp";
      const size_t payload = at + head + (type == "jxlp" ? 4 : 0);
      if (at + size > file.size() || payload > at + size) die("bad box size");
      if (is_cs) cs.insert(cs.end(), file.begin() + long(payload), file.begin() + long(at + size));
      boxes.push_back({at, size, payload, is_cs});
      at += size;
    }
  }
  // ---- one traced decode by the oracle ----
  int status = 0;
  char err[512] = {0};
  void* h = jxlo_decode(file.data(), file.size(), 0, 1, 0, &status, err, sizeof err);
  if (!h) fprintf(stderr, "%s\n", err), die("the oracle could not decode the input");
  jxlo_free(h);
  // ---- the first frame's layout ----
  ImageHeader ih;
  const size_t frame_at = parse_codestream_header(cs.data(), cs.size(), &ih);
  BitReader br(cs.data(), cs.size(), frame_at * 8);
  const FrameHeader fh = parse_frame_header(br, ih);
  const size_t toc_bit = br.pos();
  if (fh.encoding != Encoding::kVarDct) die("the first frame is not a VarDCT frame");
  const Toc toc = parse_toc(br, fh);
  if (toc.single_entry()) die("a single-section frame is not rewritten");
  if (BitReader(cs.data(), cs.size(), toc_bit).read(1)) die("a permuted TOC is not rewritten");
  const uint32_t num_lf = fh.num_lf_groups(), num_groups = fh.num_groups(), P = fh.passes.num_passes;
  if (jxlb::g_codes.size() != P) die("the HF pass codes were not traced");
  const size_t frame_end = toc.data_begin + toc.total_size;
  auto sec = [&](size_t i) { return std::make_pair(toc.entries[i].offset * 8, (toc.entries[i].offset + toc.entries[i].size) * 8); };
  // ---- tokens of every HF stream, with a representative context per cluster ----
  Lz77Counts lzc;
  std::vector<BitWriter> sections(toc.entries.size());
  std::vector<EntropyEncoder> enc(P);
  std::vector<std::vector<Sym>> syms(size_t(P) * num_groups);
  std::vector<std::vector<Token>> tokens(size_t(P) * num_groups);  // form modes
  std::vector<const jxlb::TracedStream*> streams(size_t(P) * num_groups);
  std::vector<std::vector<uint8_t>> maps(P);
  for (uint32_t p = 0; p < P; ++p) {
    const jxlb::TracedCode& code = jxlb::g_codes[p];
    if (code.lz77) die("the HF passes already have LZ77 codes");
    std::vector<uint32_t> rep(code.num_clusters, 0xffffffffu);
    for (uint32_t c = uint32_t(code.cluster_map.size()); c-- > 0;) rep[code.cluster_map[c]] = c;
    const uint32_t dist_ctx = uint32_t(code.cluster_map.size());
    std::vector<Sym> all;
    for (uint32_t g = 0; g < num_groups; ++g) {
      const auto [b, e] = sec(2 + num_lf + size_t(p) * num_groups + g);
      auto it = jxlb::g_streams.lower_bound(b);
      if (it == jxlb::g_streams.end() || it->first >= e) die("no traced HF stream in a pass group");
      streams[size_t(p) * num_groups + g] = &it->second;
      std::vector<Token> toks;
      for (const auto& [cl, v] : it->second.values) toks.push_back({rep[cl], v});
      if (form) {
        tokens[size_t(p) * num_groups + g] = toks;
        continue;
      }
      syms[size_t(p) * num_groups + g] = lz77_parse(toks, opt, dist_ctx, false, &lzc);
      all.insert(all.end(), syms[size_t(p) * num_groups + g].begin(), syms[size_t(p) * num_groups + g].end());
    }
    maps[p] = code.cluster_map;
    if (form) continue;
    maps[p].push_back(uint8_t(code.num_clusters));  // the distance context gets a cluster of its own
    if (code.num_clusters >= 255) die("too many clusters for a distance cluster of its own");
    static Lz77Header header;
    header = opt.header();
    enc[p].lz = &header;
    (void)all;
  }
  // ---- HfGlobal: everything but the pass codes as it was ----
  {
    const size_t hf = 1 + num_lf;
    BitWriter& w = sections[hf];
    size_t at = sec(hf).first;
    for (uint32_t p = 0; p < P; ++p) {
      const jxlb::TracedCode& code = jxlb::g_codes[p];
      copy_bits(w, cs, at, code.begin);
      at = code.end;
      if (form) {
        std::vector<Token> all;
        for (uint32_t g = 0; g < num_groups; ++g) all.insert(all.end(), tokens[size_t(p) * num_groups + g].begin(), tokens[size_t(p) * num_groups + g].end());
        enc[p].write_header(w, all, uint32_t(maps[p].size()), maps[p]);
        continue;
      }
      std::vector<Sym> all;
      for (uint32_t g = 0; g < num_groups; ++g) all.insert(all.end(), syms[size_t(p) * num_groups + g].begin(), syms[size_t(p) * num_groups + g].end());
      enc[p].write_header_syms(w, all, uint32_t(maps[p].size()), maps[p]);
    }
    w.pad();  // nothing follows the last pass code but padding
  }
  // ---- pass groups: the HF preset bits, the new stream, then whatever followed the old one ----
  for (uint32_t p = 0; p < P; ++p)
    for (uint32_t g = 0; g < num_groups; ++g) {
      const size_t i = 2 + num_lf + size_t(p) * num_groups + g;
      const auto [b, e] = sec(i);
      const jxlb::TracedStream& s = *streams[size_t(p) * num_groups + g];
      BitWriter& w = sections[i];
      copy_bits(w, cs, b, s.begin);
      if (form) enc[p].write_tokens(w, tokens[size_t(p) * num_groups + g]);
      else enc[p].write_syms(w, syms[size_t(p) * num_groups + g]);
      bool rest = false;  // anything but zero padding after the HF data
      for (size_t k = s.end; k < e && !rest; ++k) rest = (cs[k / 8] >> (k % 8)) & 1;
      if (rest) copy_bits(w, cs, s.end, e);
      w.pad();
    }
  for (size_t i = 0; i < 2 + num_lf; ++i)
    if (i != 1 + num_lf) {
      copy_bits(sections[i], cs, sec(i).first, sec(i).second);
    }
  // ---- codestream: headers as they were, a new TOC, the sections, anything after the frame ----
  BitWriter out;
  copy_bits(out, cs, 0, toc_bit);
  out.write(1, 0);  // not permuted
  out.pad();
  for (const BitWriter& s : sections) {
    const uint32_t sz = uint32_t(s.bytes.size());
    if (sz < 1024) write_u32(out, 0, 10, sz);
    else if (sz < 17408) write_u32(out, 1, 14, sz - 1024);
    else if (sz < 4211712) write_u32(out, 2, 22, sz - 17408);
    else write_u32(out, 3, 30, sz - 4211712);
  }
  out.pad();
  for (const BitWriter& s : sections) out.append(s);
  out.bytes.insert(out.bytes.end(), cs.begin() + long(frame_end), cs.end());
  const std::vector<uint8_t>& ncs = out.bytes;
  // ---- container: every box as it was; the codestream boxes carry the new bytes, the last one the new tail ----
  std::vector<uint8_t> res;
  if (bare) {
    res = ncs;
  } else {
    size_t taken = 0, last = 0;
    for (size_t i = 0; i < boxes.size(); ++i)
      if (boxes[i].codestream) last = i;
    for (size_t i = 0; i < boxes.size(); ++i) {
      const Box& b = boxes[i];
      if (!b.codestream) {
        res.insert(res.end(), file.begin() + long(b.at), file.begin() + long(b.at + b.size));
        continue;
      }
      size_t n = i == last ? ncs.size() - taken : b.at + b.size - b.payload;
      if (i != last && taken + n > toc_bit / 8) die("a codestream box before the last one reaches the TOC");
      const size_t head = b.payload - b.at, size = head + n;
      if (size > 0xffffffffu) die("box too large");
      const uint8_t sz[4] = {uint8_t(size >> 24), uint8_t(size >> 16), uint8_t(size >> 8), uint8_t(size)};
      res.insert(res.end(), sz, sz + 4);
      res.insert(res.end(), file.begin() + long(b.at + 4), file.begin() + long(b.payload));
      res.insert(res.end(), ncs.begin() + long(taken), ncs.begin() + long(taken + n));
      taken += n;
    }
  }
  FILE* f = fopen(argv[2], "wb");
  if (!f) die("cannot write the output");
  fwrite(res.data(), 1, res.size(), f);
  fclose(f);
  fprintf(stderr, "hf-lz77 %s: %llu values copied, %llu copies from the first value\n", opt.mode.c_str(),
          (unsigned long long)lzc.copied, (unsigned long long)lzc.from_start);
  return 0;
}
