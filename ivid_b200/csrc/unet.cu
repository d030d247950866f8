#include "unet.h"

#include <algorithm>
#include <cmath>
#include <cstring>

#include "json_min.h"

namespace ivid {

// ==================================================================================================
// config
// ==================================================================================================
static UnetConfig parse_config(const std::string& text) {
  JsonValue j;
  try {
    j = JsonParser(text).parse();
  } catch (const std::exception& e) {
    throw Error(kErrInvalidArgument, e.what());
  }
  IVID_REQUIRE(j.kind == JsonValue::kObject, "backbone config must be a JSON object");
  // accept a whole reference config file ({"backbone": {"name", "args"}, ...}), its "backbone" object, or bare args
  if (j.has("backbone") && j.at("backbone").kind == JsonValue::kObject) j = JsonValue(j.at("backbone"));
  if (j.has("args") && j.at("args").kind == JsonValue::kObject) j = JsonValue(j.at("args"));
  UnetConfig c;
  auto geti = [&](const char* k, int& dst, bool required) {
    if (j.has(k)) dst = static_cast<int>(j.at(k).num);
    else IVID_REQUIRE(!required, std::string("backbone config: missing '") + k + "'");
  };
  auto getb = [&](const char* k, bool& dst) { if (j.has(k)) dst = j.at(k).kind == JsonValue::kBool ? j.at(k).b : j.at(k).num != 0; };
  geti("image_size", c.image_size, true);
  geti("in_channels", c.in_channels, true);
  geti("model_channels", c.model_channels, true);
  geti("out_channels", c.out_channels, true);
  geti("num_res_blocks", c.num_res_blocks, true);
  IVID_REQUIRE(j.has("attention_resolutions"), "backbone config: missing 'attention_resolutions'");
  for (auto& v : j.at("attention_resolutions").arr) c.attention_resolutions.push_back(static_cast<int>(v.num));
  if (j.has("channel_mult")) {
    c.channel_mult.clear();
    for (auto& v : j.at("channel_mult").arr) c.channel_mult.push_back(v.num);
  }
  if (j.has("dropout")) c.dropout = j.at("dropout").num;
  getb("conv_resample", c.conv_resample);
  geti("num_classes", c.num_classes, false);
  getb("has_null_class", c.has_null_class);
  if (c.num_classes == 0) c.has_null_class = false;       // adm.py:350
  getb("use_fp16", c.use_fp16);
  geti("num_groups", c.num_groups, false);
  geti("num_heads", c.num_heads, false);                  // null -> keeps default (adm.py:330); unused with head channels
  geti("num_head_channels", c.num_head_channels, false);
  getb("use_scale_shift_norm", c.use_scale_shift_norm);
  getb("resblock_updown", c.resblock_updown);
  return c;
}

Unet::Unet(const std::string& cfg_json) : cfg_(parse_config(cfg_json)) { build_topology(); }

int Unet::add_param(const std::string& name, std::vector<int64_t> shape, bool is_buffer) {
  ParamSpec p;
  p.name = name;
  p.shape = std::move(shape);
  p.is_buffer = is_buffer;
  pindex_[name] = static_cast<int>(params_.size());
  params_.push_back(std::move(p));
  return static_cast<int>(params_.size()) - 1;
}

const ParamSpec& Unet::P(const std::string& name) const {
  auto it = pindex_.find(name);
  if (it == pindex_.end()) throw Error(kErrState, "internal: unknown parameter " + name);
  const ParamSpec& p = params_[it->second];
  if (!p.set) throw Error(kErrState, "parameter '" + name + "' was never set (load_state_dict incomplete)");
  return p;
}

// State-dict schema + block structure.  Follows the constructor of the reference (adm.py:356-487) layer for layer so that
// key names ("input_blocks.3.0.in_layers.0.weight", ...) and shapes match torch's registration order.
void Unet::build_topology() {
  const UnetConfig& c = cfg_;
  IVID_REQUIRE(c.in_channels <= 16, "in_channels must be <= 16");
  IVID_REQUIRE(c.num_groups >= 1 && c.num_groups <= 64, "num_groups must be in [1,64]");
  const int mc = c.model_channels;
  const int E = mc * 4;
  embed_dim_ = E;

  add_param("time_embed.0.freqs", {mc / 2}, /*is_buffer=*/true);
  add_param("time_embed.1.weight", {E, mc});
  add_param("time_embed.1.bias", {E});
  add_param("time_embed.3.weight", {E, E});
  add_param("time_embed.3.bias", {E});
  if (c.num_classes > 0) add_param("label_emb.weight", {c.num_classes, E});

  // head width of an attention block over ch channels (AttentionBlock.__init__ adm.py:266-273, QKVAttention adm.py:244)
  auto head_width = [&](int ch) {
    int hc;
    if (c.num_head_channels != -1) {
      IVID_REQUIRE(c.num_head_channels > 0 && ch % c.num_head_channels == 0,
                   "q,k,v channels " + std::to_string(ch) + " is not divisible by num_head_channels " + std::to_string(c.num_head_channels));
      hc = c.num_head_channels;
    } else {
      IVID_REQUIRE(c.num_heads > 0 && ch % c.num_heads == 0,
                   "attention channels " + std::to_string(ch) + " are not divisible by num_heads " + std::to_string(c.num_heads));
      hc = ch / c.num_heads;
    }
    if (hc % 64 != 0)
      throw Error(kErrNotImplemented, "attention head width " + std::to_string(hc) + " is not a multiple of 64 channels");
    return hc;
  };
  // Level widths: num_groups must divide each (the reference's GroupNorm32 asserts it), checked as the blocks are made.  The
  // kernels further need C % 8 == 0 (16-byte NHWC fp16 rows for TMA), checked once the whole topology stands, so that any
  // network the reference rejects still raises its AssertionError.
  std::vector<int> widths;
  auto add_res = [&](const std::string& pfx, int cin, int cout, int mode, int cat0 = 0) {
    ResBlockDef r;
    r.pfx = pfx; r.cin = cin; r.cout = cout; r.mode = mode; r.cat0 = cat0;
    IVID_REQUIRE(cin % c.num_groups == 0 && cout % c.num_groups == 0, "num_groups must divide channels");
    widths.insert(widths.end(), {cin, cout, cat0});
    add_param(pfx + ".in_layers.0.weight", {cin});
    add_param(pfx + ".in_layers.0.bias", {cin});
    add_param(pfx + ".in_layers.2.weight", {cout, cin, 3, 3});
    add_param(pfx + ".in_layers.2.bias", {cout});
    const int ew = c.use_scale_shift_norm ? 2 * cout : cout;          // adm.py:176
    add_param(pfx + ".emb_layers.1.weight", {ew, E});
    add_param(pfx + ".emb_layers.1.bias", {ew});
    add_param(pfx + ".out_layers.0.weight", {cout});
    add_param(pfx + ".out_layers.0.bias", {cout});
    add_param(pfx + ".out_layers.3.weight", {cout, cout, 3, 3});
    add_param(pfx + ".out_layers.3.bias", {cout});
    r.skip_conv = (cin != cout);
    if (r.skip_conv) {
      add_param(pfx + ".skip_connection.weight", {cout, cin, 1, 1});
      add_param(pfx + ".skip_connection.bias", {cout});
    }
    r.film_off = film_total_;
    film_total_ += ew;
    res_.push_back(r);
    return static_cast<int>(res_.size()) - 1;
  };
  auto add_attn = [&](const std::string& pfx, int ch) {
    AttnBlockDef a;
    a.pfx = pfx; a.C = ch; a.head_ch = head_width(ch);
    add_param(pfx + ".norm.weight", {ch});
    add_param(pfx + ".norm.bias", {ch});
    add_param(pfx + ".qkv.weight", {3 * ch, ch, 1});
    add_param(pfx + ".qkv.bias", {3 * ch});
    add_param(pfx + ".proj_out.weight", {ch, ch, 1});
    add_param(pfx + ".proj_out.bias", {ch});
    attn_.push_back(a);
    return static_cast<int>(attn_.size()) - 1;
  };
  auto add_resample = [&](const std::string& pfx, int ch, int mode) {
    ResampleDef r;
    r.pfx = pfx; r.C = ch; r.mode = mode; r.conv = c.conv_resample;
    widths.push_back(ch);
    if (r.conv) {
      const std::string sub = mode == 2 ? ".op" : ".conv";      // Downsample2d.op (adm.py:111) / Upsample2d.conv (adm.py:81)
      add_param(pfx + sub + ".weight", {ch, ch, 3, 3});
      add_param(pfx + sub + ".bias", {ch});
    }
    resample_.push_back(r);
    return static_cast<int>(resample_.size()) - 1;
  };
  auto in_attn = [&](int ds) {
    return std::find(c.attention_resolutions.begin(), c.attention_resolutions.end(), ds) != c.attention_resolutions.end();
  };

  int ch = static_cast<int>(c.channel_mult[0] * mc);
  const int input_ch = ch;
  in_ch_stem_ = ch;
  add_param("input_blocks.0.0.weight", {ch, c.in_channels, 3, 3});
  add_param("input_blocks.0.0.bias", {ch});
  {
    BlockDef b;
    b.is_input = true;   // the stem conv: no layers, handled explicitly
    blocks_.push_back(b);
  }
  int ds = c.image_size;
  std::vector<int> input_block_chs{ch};
  int ib = 1;
  const int levels = static_cast<int>(c.channel_mult.size());
  for (int level = 0; level < levels; ++level) {
    const int outc = static_cast<int>(c.channel_mult[level] * mc);
    for (int r = 0; r < c.num_res_blocks; ++r) {
      BlockDef b;
      b.is_input = true;
      const std::string pfx = "input_blocks." + std::to_string(ib);
      b.layers.push_back({LayerKind::kResBlock, add_res(pfx + ".0", ch, outc, 0)});
      ch = outc;
      if (in_attn(ds)) b.layers.push_back({LayerKind::kAttention, add_attn(pfx + ".1", ch)});
      blocks_.push_back(b);
      input_block_chs.push_back(ch);
      ++ib;
    }
    if (level != levels - 1) {
      BlockDef b;
      b.is_input = true;
      if (c.resblock_updown) b.layers.push_back({LayerKind::kResBlock, add_res("input_blocks." + std::to_string(ib) + ".0", ch, ch, 2)});
      else b.layers.push_back({LayerKind::kResample, add_resample("input_blocks." + std::to_string(ib) + ".0", ch, 2)});      // adm.py:409-412
      blocks_.push_back(b);
      input_block_chs.push_back(ch);
      ++ib;
      ds /= 2;
    }
  }
  {
    BlockDef b;
    b.layers.push_back({LayerKind::kResBlock, add_res("middle_block.0", ch, ch, 0)});
    b.layers.push_back({LayerKind::kAttention, add_attn("middle_block.1", ch)});
    b.layers.push_back({LayerKind::kResBlock, add_res("middle_block.2", ch, ch, 0)});
    blocks_.push_back(b);
  }
  int ob = 0;
  for (int level = levels - 1; level >= 0; --level) {
    const int outc = static_cast<int>(mc * c.channel_mult[level]);
    for (int i = 0; i <= c.num_res_blocks; ++i) {
      BlockDef b;
      b.is_output = true;
      const std::string pfx = "output_blocks." + std::to_string(ob);
      const int ich = input_block_chs.back();
      input_block_chs.pop_back();
      int li = 0;
      b.layers.push_back({LayerKind::kResBlock, add_res(pfx + "." + std::to_string(li++), ch + ich, outc, 0, ch)});
      ch = outc;
      if (in_attn(ds)) b.layers.push_back({LayerKind::kAttention, add_attn(pfx + "." + std::to_string(li++), ch)});
      if (level != 0 && i == c.num_res_blocks) {
        if (c.resblock_updown) b.layers.push_back({LayerKind::kResBlock, add_res(pfx + "." + std::to_string(li++), ch, ch, 1)});
        else b.layers.push_back({LayerKind::kResample, add_resample(pfx + "." + std::to_string(li++), ch, 1)});               // adm.py:475-478
        ds *= 2;
      }
      blocks_.push_back(b);
      ++ob;
    }
  }
  final_ch_ = ch;
  IVID_REQUIRE(ch == input_ch, "final channel count must equal the stem width (adm.py:486 uses input_ch)");
  for (int w : widths)
    if (w % 8 != 0)
      throw Error(kErrNotImplemented, "channel width " + std::to_string(w) + " is not a multiple of 8 (16-byte NHWC fp16 rows)");
  add_param("out.0.weight", {ch});
  add_param("out.0.bias", {ch});
  add_param("out.2.weight", {c.out_channels, input_ch, 3, 3});
  add_param("out.2.bias", {c.out_channels});
}

void Unet::set_param(const std::string& name, const float* data, const int64_t* shape, int ndim) {
  auto it = pindex_.find(name);
  if (it == pindex_.end()) throw Error(kErrInvalidArgument, "unexpected key in state_dict: " + name);
  ParamSpec& p = params_[it->second];
  bool same = static_cast<int>(p.shape.size()) == ndim;
  for (int i = 0; same && i < ndim; ++i) same = p.shape[i] == shape[i];
  if (!same) throw Error(kErrInvalidArgument, "size mismatch for " + name);
  p.host.assign(data, data + p.numel());
  p.set = true;
}

// ==================================================================================================
// weight packing
// ==================================================================================================
namespace {
struct ArenaBuilder {
  std::vector<uint8_t> buf;
  size_t alloc(size_t bytes) {
    const size_t off = (buf.size() + 255) & ~size_t(255);
    buf.resize(off + bytes, 0);
    return off;
  }
  template <class T> T* at(size_t off) { return reinterpret_cast<T*>(buf.data() + off); }
};

// Stem: the 64 operand channels of the packed network input are  hi | lo | hi  of a two-term fp16 split of x
// (pack_input_kernel); the matching weight columns are  Wh | Wh | Wl  with W = Wh + Wl, so that the fp16 tensor-core
// product reproduces x*W to ~2^-21 (the lo*Wl term is dropped).
void pack_stem_rows(__half* dst, int Ktot, const float* w, int cout, int cin, int cin_pad) {
  for (int co = 0; co < cout; ++co)
    for (int tap = 0; tap < 9; ++tap)
      for (int ci = 0; ci < cin; ++ci) {
        const float v = w[(static_cast<size_t>(co) * cin + ci) * 9 + tap];
        const __half hi = __float2half_rn(v);
        const __half lo = __float2half_rn(v - __half2float(hi));
        __half* row = dst + static_cast<size_t>(co) * Ktot + tap * cin_pad;
        row[ci] = hi; row[cin + ci] = hi; row[2 * cin + ci] = lo;
      }
}

// Output head as a 1x1 GEMM over 9*Co columns (column tap*Co + c holds W[c][:, tap]), split precision:
// K = [Wh | Wh | Wl] against the activation segments [a_hi | a_lo | a_hi] (GnApplyParams::out_lo), each third padded to
// Cp = conv_pad_k(C) columns.
void pack_out_rows(__half* dst, int C, int Cp, const float* w, int co_n) {
  const int K = 3 * Cp;
  for (int tap = 0; tap < 9; ++tap)
    for (int c = 0; c < co_n; ++c)
      for (int ci = 0; ci < C; ++ci) {
        const float v = w[(static_cast<size_t>(c) * C + ci) * 9 + tap];
        const __half hi = __float2half_rn(v);
        const __half lo = __float2half_rn(v - __half2float(hi));
        __half* row = dst + static_cast<size_t>(tap * co_n + c) * K;
        row[ci] = hi; row[Cp + ci] = hi; row[2 * Cp + ci] = lo;
      }
}
}  // namespace

void Unet::set_precision(int precision) {
  IVID_REQUIRE(precision == 0 || precision == 1, "precision must be 0 (fp16) or 1 (fp8 ResBlock convs)");
  precision_ = precision;
}

void Unet::finalize(int device) {
  IVID_CHECK_CUDA(cudaSetDevice(device));
  for (const auto& p : params_)
    if (!p.set) throw Error(kErrState, "parameter '" + p.name + "' was never set (load_state_dict incomplete)");
  plans_.clear();
  if (arena_) { cudaFree(arena_); arena_ = nullptr; }
  device_ = device;
  ArenaBuilder ab;
  auto put_f32 = [&](const std::vector<float>& v, size_t pad_to = 0) {
    const size_t n = std::max(v.size(), pad_to);
    const size_t off = ab.alloc(n * 4);
    std::memcpy(ab.at<float>(off), v.data(), v.size() * 4);
    return off;
  };
  auto pack_gn = [&](const std::string& pfx, int C) {
    GnW g; g.C = C;
    g.g_off = put_f32(P(pfx + ".weight").host);
    g.b_off = put_f32(P(pfx + ".bias").host);
    return g;
  };
  // conv_pack over the named parameters (other arguments as there), placed as e4m3 columns, fp16 columns, bias
  auto put_conv = [&](const std::string& wname, const std::string& bname, int cout, int cin, int pitch, int ksz,
                       const std::string& skip_w = "", const std::string& skip_b = "", int cin2 = 0, int cin2a = 0,
                       bool e4m3 = false) {
    const ConvPack pk = conv_pack(P(wname).host.data(), P(bname).host.data(), cout, cin, ksz, pitch,
                                  cin2 > 0 ? P(skip_w).host.data() : nullptr, cin2 > 0 ? P(skip_b).host.data() : nullptr,
                                  cin2, cin2a, e4m3);
    ConvW cw;
    cw.cout = cout; cw.cout_pad = pk.cout_pad; cw.K = pk.K; cw.fp8 = pk.e4m3; cw.e8 = pk.e;
    if (pk.e4m3) {
      cw.w8_off = ab.alloc(pk.w8.size());
      std::memcpy(ab.at<uint8_t>(cw.w8_off), pk.w8.data(), pk.w8.size());
    }
    if (pk.K > 0) {
      cw.w_off = ab.alloc(pk.w16.size() * 2);
      std::memcpy(ab.at<__half>(cw.w_off), pk.w16.data(), pk.w16.size() * 2);
    }
    cw.b_off = put_f32(pk.bias);
    return cw;
  };
  auto pack_lin = [&](const std::string& pfx) {
    const ParamSpec& w = P(pfx + ".weight");
    LinW l; l.O = static_cast<int>(w.shape[0]); l.K = static_cast<int>(w.shape[1]);
    l.w_off = put_f32(w.host);
    l.b_off = put_f32(P(pfx + ".bias").host);
    return l;
  };

  freqs_off_ = put_f32(P("time_embed.0.freqs").host);
  te1_ = pack_lin("time_embed.1");
  te2_ = pack_lin("time_embed.3");
  if (cfg_.num_classes > 0) label_off_ = put_f32(P("label_emb.weight").host);
  // FiLM table weights: all emb_layers.1 stacked row-wise in ResBlock creation order
  {
    film_.O = film_total_; film_.K = embed_dim_;
    film_.w_off = ab.alloc(static_cast<size_t>(film_total_) * embed_dim_ * 4);
    film_.b_off = ab.alloc(static_cast<size_t>(film_total_) * 4);
    for (const auto& r : res_) {
      const auto& w = P(r.pfx + ".emb_layers.1.weight").host;
      const auto& b = P(r.pfx + ".emb_layers.1.bias").host;
      // swizzled K-chunk-major [E/32][film_total][32] when E % 32 == 0 (see film_table_kernel), row-major otherwise
      if (embed_dim_ % 32 == 0) {
        float* dst = ab.at<float>(film_.w_off);
        const int rows_w = static_cast<int>(w.size() / embed_dim_);
        for (int o = 0; o < rows_w; ++o)
          for (int kc = 0; kc < embed_dim_; kc += 32)
            for (int g = 0; g < 8; ++g)      // 16-byte groups XOR-swizzled with the output index (film_table_kernel)
              std::memcpy(dst + (static_cast<size_t>(kc / 32) * film_total_ + r.film_off + o) * 32 + ((g ^ ((r.film_off + o) & 7)) << 2),
                          w.data() + static_cast<size_t>(o) * embed_dim_ + kc + g * 4, 16);
      } else {
        std::memcpy(ab.at<float>(film_.w_off) + static_cast<size_t>(r.film_off) * embed_dim_, w.data(), w.size() * 4);
      }
      std::memcpy(ab.at<float>(film_.b_off) + r.film_off, b.data(), b.size() * 4);
    }
  }
  in_conv_ = put_conv("input_blocks.0.0.weight", "input_blocks.0.0.bias", in_ch_stem_, cfg_.in_channels, 64, 3);
  IVID_REQUIRE(3 * cfg_.in_channels <= 64, "in_channels must be <= 21 (two-term input split inside 64 operand channels)");
  pack_stem_rows(ab.at<__half>(in_conv_.w_off), in_conv_.K, P("input_blocks.0.0.weight").host.data(), in_ch_stem_, cfg_.in_channels, 64);
  for (auto& r : resample_)
    if (r.conv) {
      const std::string sub = r.mode == 2 ? ".op" : ".conv";
      // the stride-2 conv runs as a 1x1 GEMM over the 9C im2col channels (one segment, padded at its end); the upsample
      // conv is an ordinary 3x3 conv over C channels
      r.w = put_conv(r.pfx + sub + ".weight", r.pfx + sub + ".bias", r.C, r.C, r.mode == 2 ? r.C : conv_pad_k(r.C), 3);
    }
  for (auto& r : res_) {
    r.gn1 = pack_gn(r.pfx + ".in_layers.0", r.cin);
    r.conv1 = put_conv(r.pfx + ".in_layers.2.weight", r.pfx + ".in_layers.2.bias", r.cout, r.cin, conv_pad_k(r.cin), 3,
                       "", "", 0, 0, precision_ == 1);
    r.gn2 = pack_gn(r.pfx + ".out_layers.0", r.cout);
    r.conv2 = put_conv(r.pfx + ".out_layers.3.weight", r.pfx + ".out_layers.3.bias", r.cout, r.cout, conv_pad_k(r.cout), 3,
                       r.pfx + ".skip_connection.weight", r.pfx + ".skip_connection.bias", r.skip_conv ? r.cin : 0, r.cat0,
                       precision_ == 1);
  }
  for (auto& a : attn_) {
    a.gn = pack_gn(a.pfx + ".norm", a.C);
    a.qkv = put_conv(a.pfx + ".qkv.weight", a.pfx + ".qkv.bias", 3 * a.C, a.C, conv_pad_k(a.C), 1);
    a.proj = put_conv(a.pfx + ".proj_out.weight", a.pfx + ".proj_out.bias", a.C, a.C, conv_pad_k(a.C), 1);
  }
  out_gn_ = pack_gn("out.0", final_ch_);
  out_conv_ = put_conv("out.2.weight", "out.2.bias", cfg_.out_channels, final_ch_, conv_pad_k(final_ch_), 3);
  // split-precision 1x1 form of the same conv (see pack_out_rows); bias is added by eps_gather_kernel
  out_split_ = 9 * cfg_.out_channels <= 64 && getenv("IVID_NO_OUTSPLIT") == nullptr;
  if (out_split_) {
    out1x1_.cout = 64; out1x1_.cout_pad = 64; out1x1_.K = 3 * conv_pad_k(final_ch_);
    out1x1_.w_off = ab.alloc(static_cast<size_t>(64) * out1x1_.K * 2);
    pack_out_rows(ab.at<__half>(out1x1_.w_off), final_ch_, conv_pad_k(final_ch_), P("out.2.weight").host.data(), cfg_.out_channels);
    out1x1_.b_off = put_f32(std::vector<float>(64, 0.f));
  }

  arena_bytes_ = (ab.buf.size() + 255) & ~size_t(255);
  IVID_CHECK_CUDA(cudaMalloc(&arena_, arena_bytes_));
  IVID_CHECK_CUDA(cudaMemcpy(arena_, ab.buf.data(), ab.buf.size(), cudaMemcpyHostToDevice));
}

Unet::~Unet() {
  plans_.clear();
  if (cap_stream_) cudaStreamDestroy(cap_stream_);
  if (arena_) cudaFree(arena_);
}

// ==================================================================================================
// execution plan
// ==================================================================================================
struct Plan {
  int N = 0;
  int H = 0, W = 0;        // input geometry
  AttnPerturb pert;        // normalised: row0 = N and no layers when unperturbed, layers sorted
  uint64_t last_use = 0;   // Unet::plan_uses_ at the latest forward
  uint8_t* ws = nullptr;
  size_t ws_bytes = 0;
  double* stats_base = nullptr;
  size_t stats_bytes = 0;
  struct OpRec {
    const char* label;      // kernel family (profile aggregation key)
    double flops;           // algorithmic FLOPs of this launch (tensor-core ops)
    double bytes;           // algorithmic HBM bytes of this launch (memory-bound ops)
    std::string note;       // shape description (per-op profile dump)
    std::function<void(cudaStream_t)> fn;
    int block;              // index into Unet::blocks_ of the block the op belongs to; -1: embeddings, input packing, head
  };
  std::vector<OpRec> ops;
  int op_block = -1;        // block of the ops the walk adds next
  void add_op(const char* label, double flops, double bytes, std::string note, std::function<void(cudaStream_t)> fn) {
    ops.push_back(OpRec{label, flops, bytes, std::move(note), std::move(fn), op_block});
  }
  // Feature reuse (DeepCache).  A reuse forward at branch b runs the ops of input blocks 0..b and output blocks L-1-b..L-1
  // (blocks_ indices >= n_blocks - 1 - b) and those of no block.  It reads the output of output block L-2-b, with its fp16
  // copy and its statistics, as the plan's last full forward left them.  The walk takes statistics block by block, so the
  // kept blocks' statistics are the arena's head [0, block_stats[b + 1]) and tail [block_stats[n_blocks - 1 - b], end): a
  // reuse forward zeroes only those, and the statistics of every skipped block, the cached tensor's among them, stay as the
  // last full forward left them, whatever branches ran in between.
  int n_blocks = 0;
  std::vector<size_t> block_stats;   // arena offset of the first statistics each block takes
  bool cache_valid = false;          // a full forward has been enqueued on this plan
  bool kept(int block, int branch) const {
    return branch < 0 || block < 0 || block <= branch || block >= n_blocks - 1 - branch;
  }
  // One forward: zero the statistics arena, then enqueue every op on s; branch >= 0: the reuse forward at that branch, which
  // zeroes the kept blocks' statistics and runs the kept ops only.  With `ev` (ops.size() + 1 events), ev[i] and ev[i + 1]
  // bracket op i (nothing in between for an op the reuse forward skips).
  void run(cudaStream_t s, cudaEvent_t* ev = nullptr, int branch = -1) const {
    if (branch < 0) {
      IVID_CHECK_CUDA(cudaMemsetAsync(stats_base, 0, stats_bytes, s));
    } else {
      uint8_t* base = reinterpret_cast<uint8_t*>(stats_base);
      const size_t head = block_stats[branch + 1], tail = block_stats[n_blocks - 1 - branch];
      IVID_CHECK_CUDA(cudaMemsetAsync(base, 0, head, s));
      if (tail < stats_bytes) IVID_CHECK_CUDA(cudaMemsetAsync(base + tail, 0, stats_bytes - tail, s));
    }
    if (ev) IVID_CHECK_CUDA(cudaEventRecord(ev[0], s));
    for (size_t i = 0; i < ops.size(); ++i) {
      if (kept(ops[i].block, branch)) ops[i].fn(s);
      if (ev) IVID_CHECK_CUDA(cudaEventRecord(ev[i + 1], s));
    }
  }
  std::vector<ConvLaunch*> convs;
  std::vector<AttnLaunch*> attns;
  // per-call inputs
  const float* x = nullptr; int Nx = 0; ivid_cond_t cond{}; const int64_t* t = nullptr; const int64_t* classes = nullptr;
  float* eps = nullptr;
  const HeadHook* hook = nullptr;
  const int* cond_stream_dev = nullptr;
  // CUDA graphs of the whole forward (memset + ~215 launches), one per distinct set of per-call pointers / by-value inputs:
  // the launch records bake them in, so a replay is valid exactly when the key matches.
  struct GraphKey {
    const void* x; int Nx; const void* t; const void* classes; void* eps;
    int kind; const void* y; const void* mask; const void* mask_rgb; const void* noise; uint64_t seed; uint32_t stream_id;
    const void* stream_dev;
    uint64_t hook_key;
    int sr_scale;
    int cache_branch;        // -1: full forward; b: reuse forward at branch b
    bool operator==(const GraphKey& o) const {
      return hook_key == o.hook_key && sr_scale == o.sr_scale && cache_branch == o.cache_branch && x == o.x && Nx == o.Nx && t == o.t && classes == o.classes && eps == o.eps && kind == o.kind && y == o.y && mask == o.mask &&
             mask_rgb == o.mask_rgb && noise == o.noise && seed == o.seed && stream_id == o.stream_id && stream_dev == o.stream_dev;
    }
  };
  struct GraphEntry { GraphKey key; cudaGraphExec_t exec; uint64_t last_use; };
  // named block outputs (debug taps: per-layer parity tests read them back after a forward)
  struct Tap { std::string name; const float* d32; const __half* d16; int C, H, W; };
  std::vector<Tap> taps;
  std::vector<GraphEntry> graphs;
  uint64_t runs = 0;
  uint64_t graph_hits = 0, graph_captures = 0;      // a caller whose pointers change on every call gains nothing from capturing
  ~Plan() {
    for (auto& g : graphs) cudaGraphExecDestroy(g.exec);
    for (auto* c : convs) conv_launch_destroy(c);
    for (auto* a : attns) attn_launch_destroy(a);
    if (ws) cudaFree(ws);
  }
};

namespace {
// scratch buffers of a plan, each reused by every layer that needs it
enum Slot { kIn, kA1, kA2, kXh, kXr, kH, kQkv, kCol, kPe, kE1, kEmb, kFilm, kXt, kSlots };
struct Act {          // fp32 NHWC residual-stream tensor with per-(n,channel) statistics
  float* data = nullptr;    // null when the layout keeps the tensor as fp16 only, and in the sizing pass
  __half* d16 = nullptr;    // fp16 copy written by the producing conv (operand of the next GroupNorm / 1x1 skip conv)
  double* stats = nullptr;
  bool has16 = false;       // the producing conv writes the fp16 copy
  int id = -1;              // position in creation order (index of its BlockOut)
  int C = 0, H = 0, W = 0;
};
// a block output as the sizing pass records it and the layout places it
struct BlockOut {
  int C, H, W;
  bool may16;               // the producing conv can write it as fp16 only
  bool need32 = false;      // some consumer keeps its fp32 storage
  bool only16 = false;      // layout: may16 && !need32
  size_t off16 = 0, off32 = 0;
};
}  // namespace

void Unet::check_geometry(int H, int W) const {
  const int levels = static_cast<int>(cfg_.channel_mult.size());
  const int m = 1 << (levels - 1);
  if (H <= 0 || W <= 0 || H % m != 0 || W % m != 0)
    throw Error(kErrState, "input size " + std::to_string(H) + "x" + std::to_string(W) + " is not a multiple of " + std::to_string(m) +
                               " (2^(levels-1)): the skip connections' sizes would not match after " + std::to_string(levels - 1) + " downsamplings");
}

Plan* Unet::get_plan(int N, int H, int W, const AttnPerturb& pert) {
  Plan* found = nullptr;
  for (auto& p : plans_)
    if (p->N == N && p->H == H && p->W == W && p->pert.row0 == pert.row0 && p->pert.layers == pert.layers) found = p.get();
  if (found == nullptr) {
    check_geometry(H, W);
    if (plans_.size() >= 4) {
      IVID_CHECK_CUDA(cudaDeviceSynchronize());     // the evicted plan's workspace may still be in use by queued kernels
      plans_.erase(plans_.begin());
    }
    plans_.emplace_back(build_plan(N, H, W, pert));
    found = plans_.back().get();
  }
  found->last_use = ++plan_uses_;
  return found;
}

Plan* Unet::build_plan(int N, int SH, int SW, const AttnPerturb& pert) {
  std::unique_ptr<Plan> plan(new Plan());
  plan->N = N;
  plan->pert = pert;
  std::vector<bool> perturbed(attn_.size(), false);
  for (int i : pert.layers) perturbed[i] = true;
  plan->H = SH; plan->W = SW;
  plan->n_blocks = static_cast<int>(blocks_.size());
  plan->block_stats.assign(blocks_.size(), 0);      // block 0, the stem, takes the first statistics
  Plan* pl = plan.get();
  const int G = cfg_.num_groups;
  const float eps = 1e-5f;
  auto W8 = [&](size_t off) { return arena_ + off; };
  auto Wf = [&](size_t off) { return reinterpret_cast<const float*>(arena_ + off); };
  // a packed conv's operands (Unet::finalize) as a ConvDesc's weights, output width and bias
  auto bind = [&](ConvDesc& d, const ConvW& w) {
    d.weight = w.K > 0 ? W8(w.w_off) : nullptr;
    d.weight8 = w.fp8 ? W8(w.w8_off) : nullptr;
    d.acc_scale = std::ldexp(1.0f, -w.e8);
    d.cout_pad = w.cout_pad; d.cout = w.cout; d.bias = Wf(w.b_off);
  };

  // One walk over the topology, run twice.  The sizing pass (base == nullptr) creates no ops: it records the largest
  // request made of each scratch slot, the shape and storage needs of each block output, and the statistics bytes.  The
  // layout then places them, and the create pass (base = the workspace) walks again with real pointers, builds the
  // launches and checks every scratch and statistics request against what the layout gave it.
  size_t slot_bytes[kSlots] = {}, slot_off[kSlots] = {};
  std::vector<BlockOut> outs;
  size_t stats_bytes = 0, stats_off = 0;
  auto walk = [&](uint8_t* base) {
    const bool create = base != nullptr;
    auto scratch = [&](Slot s, size_t bytes) -> void* {
      if (!create) { slot_bytes[s] = std::max(slot_bytes[s], bytes); return nullptr; }
      IVID_REQUIRE(bytes <= slot_bytes[s], "internal: scratch request exceeds its slot");
      return base + slot_off[s];
    };
    // N x H x W x C elements of a slot
    auto s16 = [&](Slot s, int H, int Wd, int C) { return scratch(s, static_cast<size_t>(N) * H * Wd * C * 2); };
    auto s32 = [&](Slot s, int H, int Wd, int C) { return static_cast<float*>(scratch(s, static_cast<size_t>(N) * H * Wd * C * 4)); };
    // conv operand: fp16, or e4m3 (one byte per element) for a conv packed fp8
    auto sop = [&](Slot s, int H, int Wd, int C, bool e4m3) { return scratch(s, static_cast<size_t>(N) * H * Wd * C * (e4m3 ? 1 : 2)); };
    size_t soff = 0;
    auto take_stats = [&](int C) -> double* {
      const size_t o = soff;
      soff += (static_cast<size_t>(N) * C * 16 + 255) & ~size_t(255);
      if (!create) return nullptr;
      IVID_REQUIRE(soff <= stats_bytes, "internal: statistics request exceeds the arena");
      return reinterpret_cast<double*>(base + stats_off + o);
    };
    int next_id = 0;
    // may16: the producer's epilogue has no residual add, so it could write the output as fp16 only
    auto new_act = [&](int C, int H, int Wd, bool may16) {
      Act a; a.C = C; a.H = H; a.W = Wd;
      a.id = next_id++;
      a.has16 = conv_can_out16(C);
      if (!create) {
        outs.push_back(BlockOut{C, H, Wd, may16 && a.has16 && conv_can_fuse_stats(H, Wd)});
      } else {
        IVID_REQUIRE(a.id < static_cast<int>(outs.size()) && outs[a.id].C == C && outs[a.id].H == H && outs[a.id].W == Wd,
                     "internal: block output differs from the sizing pass");
        const BlockOut& o = outs[a.id];
        if (a.has16) a.d16 = reinterpret_cast<__half*>(base + o.off16);
        if (!o.only16) a.data = reinterpret_cast<float*>(base + o.off32);
      }
      a.stats = take_stats(C);
      return a;
    };
    auto use32 = [&](const Act& a) -> const float* {
      if (!create) outs[a.id].need32 = true;
      else IVID_REQUIRE(a.data != nullptr, "internal: fp32 tensor was not materialised");
      return a.data;
    };
    // ResBlocks and the output head keep the fp32 storage of their inputs even where they read the fp16 copies, so only an
    // output that a resampling conv alone reads is written as fp16 only.  Storing more outputs as fp16 only would change
    // their convs' epilogues and take their statistics from the rounded values: a change of results, not of layout.
    auto keep32 = [&](const Act& a) { use32(a); };
    // a block output as the conv's output: fp32 NHWC plus the fp16 copy, or fp16 only where the layout gave it no fp32
    auto write_to = [&](ConvDesc& d, const Act& a) {
      if (a.data != nullptr) { d.out = a.data; d.out16 = a.d16; d.out_mode = 0; }
      else { d.out = a.d16; d.out_mode = 1; }
      d.ldc = a.C; d.N = N; d.H = a.H; d.W = a.W;
    };
    // GroupNorm statistics of the output are accumulated in the conv epilogue whenever the tile geometry allows; otherwise
    // a separate pass reads the fp32 NHWC output right after the conv
    auto add_conv = [&](ConvDesc d, const Act* stats_of = nullptr, double k_alg = 0.0, double n_alg = 0.0) {
      if (!create) return;
      const bool fused = stats_of != nullptr && conv_can_fuse_stats(d.H, d.W);
      if (fused) d.stats = stats_of->stats;
      ConvLaunch* l = conv_launch_create(d);
      pl->convs.push_back(l);
      // ALGORITHMIC work: operand padding (stem: 9*Cin of 9*64 columns) and split-precision segments do not count
      const double K = k_alg > 0.0 ? k_alg : static_cast<double>(d.taps0) * d.C0 + (d.C1 > 0 ? static_cast<double>(d.taps1) * d.C1 : 0.0) +
                       (d.C2 > 0 ? static_cast<double>(d.taps2) * d.C2 : 0.0);
      const double M = static_cast<double>(d.N) * d.H * d.W;
      const double Nalg = n_alg > 0.0 ? n_alg : static_cast<double>(d.cout);
      static const char* names[2][3] = {{"conv_gemm<16>", "conv_gemm<64>", "conv_gemm<128>"},
                                        {"conv_gemm<16,e4m3>", "conv_gemm<64,e4m3>", "conv_gemm<128,e4m3>"}};
      const int bn = conv_launch_bn(l);
      const bool a8 = conv_launch_a8(l);
      const double K0 = static_cast<double>(d.taps0) * d.C0;     // bytes per element of segment 0's operands: 1 under a8
      pl->add_op(names[a8 ? 1 : 0][bn == 128 ? 2 : bn == 64 ? 1 : 0], 2.0 * M * K * Nalg,
                 M * (d.C0 * (a8 ? 1 : 2) + (d.C1 + d.C2) * 2) + M * d.cout * ((d.out_mode == 1 ? 2 : 4) + (d.out16 ? 2 : 0) + (d.residual ? 4 : 0)) +
                     (a8 ? K0 + 2 * (K - K0) : 2 * K) * d.cout_pad,
                 std::to_string(d.H) + "x" + std::to_string(d.W) + " " + std::to_string(d.C0) + (d.C1 ? "+" + std::to_string(d.C1) : "") + (d.C2 ? "+" + std::to_string(d.C2) : "") +
                     "->" + std::to_string(d.cout) + " k" + std::to_string(d.taps0) + (d.residual ? " res" : "") + (d.stats ? " stats" : "") +
                     (d.out_mode == 1 ? " f16" : "") + (d.out16 ? " +f16" : ""),
                 [l](cudaStream_t s) { conv_launch_run(l, s); });
      if (stats_of != nullptr && !fused) {
        const float* x = stats_of->data; double* st = stats_of->stats;
        IVID_REQUIRE(x != nullptr, "internal: statistics pass over a tensor without fp32 storage");
        const int HW = stats_of->H * stats_of->W, C = stats_of->C;
        pl->add_op("gn_stats", 0, static_cast<double>(N) * HW * C * 4, "", [=](cudaStream_t s) { launch_gn_stats(x, st, N, HW, C, s); });
      }
    };

    // ---- embeddings ----
    pl->op_block = -1;
    float* s_pe = s32(kPe, 1, 1, cfg_.model_channels);
    float* s_e1 = s32(kE1, 1, 1, embed_dim_);
    float* s_emb = s32(kEmb, 1, 1, embed_dim_);
    float* s_film = s32(kFilm, 1, 1, film_total_);
    float* s_xt = static_cast<float*>(scratch(kXt, static_cast<size_t>((N + 31) / 32) * embed_dim_ * 32 * 4));
    if (create) {
      const float* freqs = Wf(freqs_off_);
      const int half = cfg_.model_channels / 2, mc = cfg_.model_channels, E = embed_dim_;
      const float *w1 = Wf(te1_.w_off), *b1 = Wf(te1_.b_off), *w2 = Wf(te2_.w_off), *b2 = Wf(te2_.b_off);
      const float* lab = cfg_.num_classes > 0 ? Wf(label_off_) : nullptr;
      const float *wf = Wf(film_.w_off), *bf = Wf(film_.b_off);
      const int FT = film_total_;
      pl->add_op("embed", 2.0 * N * E * (mc + E), 4.0 * E * (mc + E), "posenc+time_embed", [=](cudaStream_t s) {
        launch_posenc(pl->t, N, freqs, half, s_pe, N, s);
        launch_linear(s_pe, w1, b1, s_e1, N, mc, E, 0, nullptr, nullptr, 1, s);
        launch_linear(s_e1, w2, b2, s_emb, N, E, E, 1, pl->classes ? lab : nullptr, pl->classes, N, s);
      });
      pl->taps.push_back({"emb", s_emb, nullptr, E, 1, 1});                 // time (+ class) embedding [N, E] (adm.py:545-555)
      pl->taps.push_back({"film", s_film, nullptr, FT, 1, 1});              // all emb_layers outputs [N, sum 2*Cout] (adm.py:174-177, 214)
      pl->add_op("embed", 2.0 * N * E * FT, 4.0 * E * FT, "film table O=" + std::to_string(FT), [=](cudaStream_t s) {
        if (E % 32 == 0) launch_film_table(s_emb, wf, bf, s_xt, s_film, N, E, FT, s);
        else launch_linear(s_emb, wf, bf, s_film, N, E, FT, 1, nullptr, nullptr, 1, s);
      });
    }
    // GroupNorm (+ FiLM from column film_off of the table; -1: none) of a0 [| a1]; the coefficients are computed in the
    // prologue of the apply kernel.  d carries the source pointers (fp32 or the fp16 copies), the geometry and the outputs.
    auto add_gn = [&](GnApplyDesc d, const Act& a0, const Act* a1, const GnW& g, int film_off) {
      if (!create) return;
      d.stats0 = a0.stats; d.stats1 = a1 ? a1->stats : nullptr;
      d.groups = G; d.eps = eps;
      d.gamma = Wf(g.g_off); d.beta = Wf(g.b_off);
      d.film = film_off >= 0 ? s_film : nullptr;
      d.film_ld = film_total_; d.film_off = std::max(film_off, 0);
      d.film_add = film_off >= 0 && !cfg_.use_scale_shift_norm;
      const int Ho = d.mode == 1 ? d.H * 2 : (d.mode == 2 ? d.H / 2 : d.H);
      const int Wo = d.mode == 1 ? d.W * 2 : (d.mode == 2 ? d.W / 2 : d.W);
      const double in_el = static_cast<double>(d.N) * d.H * d.W * (d.C0 + d.C1);
      const double out_el = static_cast<double>(d.N) * Ho * Wo * (d.C0 + d.C1);
      pl->add_op("gn_apply", 0, in_el * (d.x0_half ? 2 : 4) + out_el * (d.out_e4m3 ? 1 : 2) + (d.out_raw16 ? out_el * 2 : 0) + (d.out_raw32 ? out_el * 4 : 0),
                 std::to_string(d.H) + "x" + std::to_string(d.W) + " C" + std::to_string(d.C0) + (d.C1 ? "+" + std::to_string(d.C1) : "") +
                     " m" + std::to_string(d.mode) + (d.x0_half ? " h16" : "") + (d.out_raw16 ? " raw16" : "") + (d.out_raw32 ? " raw32" : "") +
                     (d.out_e4m3 ? " e4m3" : ""),
                 [d](cudaStream_t s) { launch_gn_apply(d, s); });
    };

    // ---- stem ----
    void* s_in = s16(kIn, SH, SW, 64);
    if (create) {
      const int Cin = cfg_.in_channels, HW = SH * SW;
      pl->add_op("pack_input", 0, static_cast<double>(N) * HW * (Cin * 4 + 128), "", [=](cudaStream_t s) {
        if (pl->cond.kind == 0) {
          launch_pack_input(pl->x, s_in, N, pl->Nx, Cin, HW, s);
        } else {
          CondPackDesc cp;
          cp.x = pl->x; cp.y = pl->cond.y_dev; cp.mask = pl->cond.mask_dev; cp.mask_rgb = pl->cond.mask_rgb_dev;
          cp.noise = pl->cond.noise_dev; cp.out = s_in; cp.N = N; cp.Nx = pl->Nx; cp.H = SH; cp.W = SW;
          cp.kind = pl->cond.kind; cp.seed = pl->cond.seed; cp.stream = pl->cond.stream_id; cp.stream_dev = pl->cond_stream_dev;
          cp.scale = pl->cond.sr_scale > 0 ? pl->cond.sr_scale : 2;
          launch_cond_pack(cp, s);
        }
      });
    }
    pl->op_block = 0;
    Act cur = new_act(in_ch_stem_, SH, SW, true);
    {
      ConvDesc d;
      d.act0 = s_in; d.C0 = 64; d.taps0 = 9;
      bind(d, in_conv_);
      write_to(d, cur);
      add_conv(d, &cur, 9.0 * cfg_.in_channels);
      if (create) pl->taps.push_back({"input_blocks.0.0", cur.data, cur.d16, cur.C, cur.H, cur.W});
    }
    std::vector<Act> skips;
    skips.push_back(cur);

    auto run_res = [&](const ResBlockDef& r, const Act& x0, const Act* x1) -> Act {
      const int Cin = x0.C + (x1 ? x1->C : 0);
      IVID_REQUIRE(Cin == r.cin, "internal: ResBlock input width mismatch at " + r.pfx);
      keep32(x0);
      if (x1) keep32(*x1);
      const int H = x0.H, Wd = x0.W;
      const int Ho = r.mode == 1 ? H * 2 : (r.mode == 2 ? H / 2 : H);
      const int Wo = r.mode == 1 ? Wd * 2 : (r.mode == 2 ? Wd / 2 : Wd);
      const bool identity = !r.skip_conv;
      // nearest-2x upsample of the identity skip is applied by the conv epilogue itself when the tile geometry allows it
      const bool res_up = identity && r.mode == 1 && x1 == nullptr && conv_can_res_up(Wo, r.cout);
      const bool need_xr = identity && (r.mode != 0 || x1 != nullptr) && !res_up;   // resampled / concatenated identity skip
      // GN1 + SiLU (+ resample) -> a1 ; raw fp16 copy for the 1x1 skip conv ; raw fp32 for resampled identity skip
      GnApplyDesc g1;
      // same-resolution blocks read the fp16 copies their producers wrote (half the GroupNorm read traffic, and the 1x1 skip
      // conv takes them directly as K segments: no raw copy pass)
      const bool use16 = r.mode == 0 && !need_xr && x0.has16 && (x1 == nullptr || x1->has16);
      if (use16) { g1.x0 = x0.d16; g1.x1 = x1 ? x1->d16 : nullptr; g1.x0_half = true; }
      else { g1.x0 = use32(x0); g1.x1 = x1 ? use32(*x1) : nullptr; }
      g1.C0 = x0.C; g1.C1 = x1 ? x1->C : 0;
      g1.N = N; g1.H = H; g1.W = Wd; g1.mode = r.mode; g1.silu = 1;
      IVID_REQUIRE(!(r.skip_conv && r.mode != 0), "internal: up/down ResBlocks keep the channel count");
      void* a1 = sop(kA1, Ho, Wo, r.cin, r.conv1.fp8);
      void* xh = r.skip_conv && !use16 ? s16(kXh, H, Wd, r.cin) : nullptr;
      float* xr = need_xr ? s32(kXr, Ho, Wo, r.cin) : nullptr;
      g1.out_act = a1; g1.out_raw16 = xh; g1.out_raw32 = xr; g1.out_e4m3 = r.conv1.fp8;
      add_gn(g1, x0, x1, r.gn1, -1);
      // conv1 -> h ; stats.  The hidden tensor only feeds GroupNorm 2: stored as fp16 (half the epilogue and GN traffic);
      // its statistics are taken from the rounded values in the conv epilogue.  Tiny feature maps keep the fp32 +
      // stats-kernel path.
      const bool h_half = conv_can_fuse_stats(Ho, Wo);
      Act h; h.C = r.cout; h.H = Ho; h.W = Wo;
      h.data = static_cast<float*>(scratch(kH, static_cast<size_t>(N) * Ho * Wo * r.cout * (h_half ? 2 : 4)));
      h.stats = take_stats(r.cout);
      {
        ConvDesc d;
        d.act0 = a1; d.C0 = r.cin; d.taps0 = 9;
        bind(d, r.conv1);
        d.out = h.data; d.ldc = r.cout; d.out_mode = h_half ? 1 : 0; d.N = N; d.H = Ho; d.W = Wo;
        add_conv(d, &h);
      }
      // GN2 * (1+scale) + shift, SiLU -> a2
      void* a2 = sop(kA2, Ho, Wo, r.cout, r.conv2.fp8);
      GnApplyDesc g2;
      g2.x0 = h.data; g2.x0_half = h_half; g2.C0 = r.cout; g2.N = N; g2.H = Ho; g2.W = Wo; g2.mode = 0; g2.silu = 1;
      g2.out_act = a2; g2.out_e4m3 = r.conv2.fp8;
      add_gn(g2, h, nullptr, r.gn2, r.film_off);
      // conv2 (+ 1x1 skip as extra K) + residual -> out
      Act out = new_act(r.cout, Ho, Wo, !identity);
      {
        ConvDesc d;
        d.act0 = a2; d.C0 = r.cout; d.taps0 = 9;
        if (r.skip_conv && use16) {
          d.act1 = x0.d16; d.C1 = x0.C; d.taps1 = 1;
          if (x1 != nullptr) { d.act2 = x1->d16; d.C2 = x1->C; d.taps2 = 1; }
        } else if (r.skip_conv) {
          // one segment over the raw concat: the packed skip columns (one segment per concat part) only line up when the
          // first part fills whole 64-channel chunks
          IVID_REQUIRE(r.cat0 % 64 == 0, "internal: raw-copy skip conv over a concat whose first part is not a multiple of 64");
          d.act1 = xh; d.C1 = r.cin; d.taps1 = 1;
        }
        bind(d, r.conv2);
        if (identity) { d.residual = need_xr ? xr : use32(x0); d.ldr = r.cout; d.residual_up = res_up; }
        write_to(d, out);
        add_conv(d, &out);
      }
      if (create) pl->taps.push_back({r.pfx, out.data, out.d16, out.C, out.H, out.W});
      return out;
    };
    auto run_attn = [&](const AttnBlockDef& a, int idx, const Act& x) -> Act {
      IVID_REQUIRE(x.C == a.C, "internal: attention width mismatch at " + a.pfx);
      const int T = x.H * x.W;
      void* a1 = s16(kA1, x.H, x.W, a.C);
      void* qkv = s16(kQkv, x.H, x.W, 3 * a.C);
      void* a2 = s16(kA2, x.H, x.W, a.C);
      GnApplyDesc g;
      if (x.has16) { g.x0 = x.d16; g.x0_half = true; } else g.x0 = use32(x);
      g.C0 = a.C; g.N = N; g.H = x.H; g.W = x.W; g.mode = 0; g.silu = 0; g.out_act = a1;
      add_gn(g, x, nullptr, a.gn, -1);
      {
        ConvDesc d;
        d.act0 = a1; d.C0 = a.C; d.taps0 = 1;
        bind(d, a.qkv);
        d.out = qkv; d.ldc = 3 * a.C; d.out_mode = 1; d.N = N; d.H = x.H; d.W = x.W;
        add_conv(d);
      }
      if (create) {
        // PAG: rows [row0, N) of a perturbed layer take the identity map (their own op); the softmax op covers the rest
        const int row0 = perturbed[idx] ? pert.row0 : N;
        AttnLaunch* l = attn_launch_create(qkv, N, T, a.C, a.head_ch, a2, row0);
        pl->attns.push_back(l);
        const std::string shape = "T=" + std::to_string(T) + " heads=" + std::to_string(a.C / a.head_ch) + " d=" + std::to_string(a.head_ch);
        if (row0 > 0)
          pl->add_op("attention", 4.0 * row0 * static_cast<double>(T) * T * a.C, static_cast<double>(row0) * T * a.C * 8, shape,
                     [l](cudaStream_t s) { attn_launch_run_softmax(l, s); });
        if (row0 < N)
          pl->add_op("attention_identity", 0, static_cast<double>(N - row0) * T * a.C * 4, shape + " rows=" + std::to_string(N - row0),
                     [l](cudaStream_t s) { attn_launch_run_identity(l, s); });
      }
      Act out = new_act(a.C, x.H, x.W, false);
      {
        ConvDesc d;
        d.act0 = a2; d.C0 = a.C; d.taps0 = 1;
        bind(d, a.proj);
        d.residual = use32(x); d.ldr = a.C;
        write_to(d, out);
        add_conv(d, &out);
      }
      if (create) pl->taps.push_back({a.pfx, out.data, out.d16, out.C, out.H, out.W});
      return out;
    };

    // plain Downsample2d / Upsample2d (resblock_updown=False): the raw block output is the conv operand (no norm in between)
    auto run_resample = [&](const ResampleDef& r, const Act& x) -> Act {
      IVID_REQUIRE(x.C == r.C, "internal: resampling layer width mismatch at " + r.pfx);
      const int Ho = r.mode == 1 ? x.H * 2 : x.H / 2, Wo = r.mode == 1 ? x.W * 2 : x.W / 2;
      Act out = new_act(r.C, Ho, Wo, false);
      const int H = x.H, Wd = x.W, C = r.C;
      if (r.conv) {
        IVID_REQUIRE(x.has16, "internal: resampling conv needs the fp16 copy of its input");
        const void* x16 = x.d16;
        ConvDesc d;
        if (r.mode == 2) {
          void* col = s16(kCol, Ho, Wo, 9 * C);           // im2col operand of the stride-2 Downsample2d conv
          if (create)
            pl->add_op("resample", 0, static_cast<double>(N) * Ho * Wo * 9 * C * 4, "im2col s2 " + std::to_string(H) + "x" + std::to_string(Wd) + " C" + std::to_string(C),
                       [=](cudaStream_t s) { launch_im2col_s2(x16, col, N, H, Wd, C, s); });
          d.act0 = col; d.C0 = 9 * C; d.taps0 = 1;
        } else {
          void* up = s16(kA1, Ho, Wo, C);
          if (create)
            pl->add_op("resample", 0, static_cast<double>(N) * Ho * Wo * C * 2.5, "nearest 2x " + std::to_string(H) + "x" + std::to_string(Wd) + " C" + std::to_string(C),
                       [=](cudaStream_t s) { launch_upsample2x_h16(x16, up, N, H, Wd, C, s); });
          d.act0 = up; d.C0 = C; d.taps0 = 9;
        }
        bind(d, r.w);
        write_to(d, out);
        add_conv(d, &out, 9.0 * C);
      } else {
        const float* src = use32(x);
        if (create) {
          float* dst = out.data; void* dst16 = out.d16; double* st = out.stats;
          const int mode = r.mode;
          pl->add_op("resample", 0, static_cast<double>(N) * (H * Wd + Ho * Wo * 1.5) * C * 4, (mode == 1 ? "nearest 2x f32 " : "avgpool f32 ") + std::to_string(H) + "x" + std::to_string(Wd),
                     [=](cudaStream_t s) { launch_resample_f32(src, dst, dst16, N, H, Wd, C, mode, s); });
          pl->add_op("gn_stats", 0, static_cast<double>(N) * Ho * Wo * C * 4, "", [=](cudaStream_t s) { launch_gn_stats(dst, st, N, Ho * Wo, C, s); });
        }
      }
      if (create) pl->taps.push_back({r.pfx, out.data, out.d16, out.C, out.H, out.W});
      return out;
    };

    for (size_t bi = 1; bi < blocks_.size(); ++bi) {
      const BlockDef& b = blocks_[bi];
      if (create) pl->block_stats[bi] = soff;
      pl->op_block = static_cast<int>(bi);
      bool first = true;
      for (const auto& l : b.layers) {
        switch (l.kind) {
          case LayerKind::kResBlock:
            if (b.is_output && first) {
              Act sk = skips.back();
              skips.pop_back();
              cur = run_res(res_[l.idx], cur, &sk);
            } else {
              cur = run_res(res_[l.idx], cur, nullptr);
            }
            break;
          case LayerKind::kAttention: cur = run_attn(attn_[l.idx], l.idx, cur); break;
          case LayerKind::kResample: cur = run_resample(resample_[l.idx], cur); break;
        }
        first = false;
      }
      if (b.is_input) skips.push_back(cur);
    }
    IVID_REQUIRE(skips.empty(), "internal: skip stack not consumed");

    // ---- output head: GN + SiLU + conv3x3 -> eps (fp32 NCHW) ----
    pl->op_block = -1;
    keep32(cur);
    const bool split_head = out_split_ && cur.has16;
    void* a1 = s16(kA1, SH, SW, cur.C);
    void* a2 = split_head ? s16(kA2, SH, SW, cur.C) : nullptr;
    GnApplyDesc go;
    if (cur.has16) { go.x0 = cur.d16; go.x0_half = true; } else go.x0 = use32(cur);
    go.C0 = cur.C; go.N = N; go.H = SH; go.W = SW; go.mode = 0; go.silu = 1; go.out_act = a1; go.out_lo = a2;
    add_gn(go, cur, nullptr, out_gn_, -1);
    if (split_head) {
      // 1x1 GEMM over 9*Co tap columns on [a_hi | a_lo | a_hi] x [Wh | Wh | Wl], then shift-and-add + bias (eps_gather_kernel):
      // each activation element is read once instead of nine times, and the product carries ~21 mantissa bits
      float* Y = s32(kH, SH, SW, 64);
      ConvDesc d;
      d.act0 = a1; d.C0 = cur.C; d.taps0 = 1;
      d.act1 = a2; d.C1 = cur.C; d.taps1 = 1;
      d.act2 = a1; d.C2 = cur.C; d.taps2 = 1;
      bind(d, out1x1_);
      d.out = Y; d.ldc = 64; d.out_mode = 0; d.N = N; d.H = SH; d.W = SW;
      add_conv(d, nullptr, 9.0 * cur.C, static_cast<double>(cfg_.out_channels));
      if (create) {
        const float* ob = Wf(out_conv_.b_off);
        const int Co = cfg_.out_channels;
        pl->add_op("eps_gather", 0, static_cast<double>(N) * SH * SW * (9.0 * Co * 4 + Co * 4), "", [=](cudaStream_t s) {
          if (pl->hook != nullptr) pl->hook->launch(Y, ob, N, SH, SW, Co, 64, s);
          else launch_eps_gather(Y, ob, pl->eps, N, SH, SW, Co, 64, s);
        });
      }
    } else if (create) {
      ConvDesc d;
      d.act0 = a1; d.C0 = cur.C; d.taps0 = 9;
      bind(d, out_conv_);
      d.out = nullptr; d.ldc = 0; d.out_mode = 2; d.N = N; d.H = SH; d.W = SW;
      ConvLaunch* l = conv_launch_create(d);
      pl->convs.push_back(l);
      // eps pointer is a per-call input: patched through the plan at run time
      pl->add_op("conv_gemm<16>", 2.0 * N * SH * SW * 9.0 * cur.C * cfg_.out_channels,
                 static_cast<double>(N) * SH * SW * (cur.C * 2 + cfg_.out_channels * 4), "",
                 [l, pl](cudaStream_t s) { conv_launch_run_out(l, pl->eps, s); });
    }
    if (!create) stats_bytes = soff;
  };

  walk(nullptr);
  // layout: statistics, scratch slots, then block outputs in creation order, each 1024-byte aligned
  size_t total = 0;
  auto place = [&](size_t bytes) {
    const size_t off = (total + 1023) & ~size_t(1023);
    total = off + bytes;
    return off;
  };
  stats_off = place(stats_bytes);
  for (int s = 0; s < kSlots; ++s) slot_off[s] = place(slot_bytes[s]);
  for (auto& o : outs) {
    const size_t n = static_cast<size_t>(N) * o.H * o.W * o.C;
    if (conv_can_out16(o.C)) o.off16 = place(n * 2);
    o.only16 = o.may16 && !o.need32;
    if (!o.only16) o.off32 = place(n * 4);
  }
  IVID_CHECK_CUDA(cudaMalloc(&pl->ws, total + 4096));
  pl->ws_bytes = total;
  pl->stats_base = reinterpret_cast<double*>(pl->ws + stats_off);
  pl->stats_bytes = stats_bytes;
  walk(pl->ws);
  return plan.release();
}

bool Unet::can_fuse_head(int W) const {
  return out_split_ && conv_can_out16(final_ch_) && cfg_.out_channels == 4 && W % 4 == 0;
}

void Unet::forward(const float* x, int Nx, int H, int W, const ivid_cond_t* cond, const int64_t* t, const int64_t* classes,
                   float* eps, int N, cudaStream_t stream, const HeadHook* hook, int cache_branch, const AttnPerturb* pert) {
  if (!finalized()) throw Error(kErrState, "AdmUnet2d: forward before .cuda()/finalize");
  IVID_REQUIRE(cache_branch >= -1 && cache_branch <= cfg_.num_res_blocks,
               "cache_branch must be in [0, num_res_blocks] = [0, " + std::to_string(cfg_.num_res_blocks) + "]");
  check_geometry(H, W);
  IVID_REQUIRE(N >= 1 && Nx >= 1 && N % Nx == 0, "forward: N must be a positive multiple of Nx");
  // reference: "this model is not class-conditioned" (adm.py:540)
  IVID_REQUIRE(classes == nullptr || cfg_.num_classes > 0, "this model is not class-conditioned");
  IVID_CHECK_CUDA(cudaSetDevice(device_));
  ivid_cond_t cnd = cond ? *cond : ivid_cond_t{};
  const int expect_in = cnd.kind == 1 ? (cnd.mask_rgb_dev ? 10 : 9) : (cnd.kind == 2 ? 8 : cfg_.in_channels);
  IVID_REQUIRE(expect_in == cfg_.in_channels, "forward: conditional inputs do not match the model's in_channels");
  IVID_REQUIRE(hook == nullptr || can_fuse_head(W), "forward: a head hook needs the tap-column output head");
  IVID_REQUIRE(cnd.kind != 2 || (cnd.sr_scale >= 0 && H % std::max(cnd.sr_scale, 1) == 0 && W % std::max(cnd.sr_scale, 1) == 0),
               "forward: the super-resolution scale must divide the input size");
  IVID_REQUIRE(hook != nullptr || eps != nullptr, "forward: eps output missing");
  AttnPerturb pt;
  pt.row0 = N;
  if (pert != nullptr && !pert->layers.empty()) {
    IVID_REQUIRE(pert->row0 >= 0 && pert->row0 <= N, "forward: the perturbed-row start must lie in [0, N]");
    pt.layers = pert->layers;
    std::sort(pt.layers.begin(), pt.layers.end());
    for (size_t i = 0; i < pt.layers.size(); ++i) {
      IVID_REQUIRE(pt.layers[i] >= 0 && pt.layers[i] < num_attention_layers(),
                   "forward: attention layer index " + std::to_string(pt.layers[i]) + " out of range [0, " +
                       std::to_string(num_attention_layers()) + ")");
      IVID_REQUIRE(i == 0 || pt.layers[i] != pt.layers[i - 1], "forward: an attention layer is listed twice");
    }
    pt.row0 = pert->row0;
    if (pt.row0 == N) pt.layers.clear();
  }

  Plan* pl = get_plan(N, H, W, pt);
  if (cache_branch >= 0 && !pl->cache_valid)
    throw Error(kErrState, "reuse forward: no full forward of this batch size and input size has run since the plan was built");
  pl->x = x; pl->Nx = Nx; pl->t = t; pl->classes = classes; pl->eps = eps;
  pl->cond = cnd;
  pl->cond_stream_dev = cond_stream_dev_;
  pl->hook = hook;
  if (cache_branch < 0) pl->cache_valid = true;      // the full forward is enqueued below
  if (!profile_) {
    // The first call of a plan runs eagerly (one-time function attributes, module loading); from the second call on the
    // forward is ONE cudaGraphLaunch.  Graphs are captured on a private stream (the caller's may be the legacy default
    // stream, which cannot be captured) and launched on the caller's stream.
    static const bool graphs_on = getenv("IVID_NO_GRAPH") == nullptr;
    ++pl->runs;
    if (graphs_on && pl->runs > 1) {
      const Plan::GraphKey key{x, Nx, t, classes, eps, cnd.kind, cnd.y_dev, cnd.mask_dev, cnd.mask_rgb_dev, cnd.noise_dev,
                               cnd.kind != 0 ? cnd.seed : 0ull, cnd.kind != 0 ? cnd.stream_id : 0u, cond_stream_dev_,
                               hook ? hook->key : 0ull, cnd.kind == 2 ? cnd.sr_scale : 0, cache_branch};
      for (auto& g : pl->graphs)
        if (g.key == key) {
          g.last_use = pl->runs;
          ++pl->graph_hits;
          IVID_CHECK_CUDA(cudaGraphLaunch(g.exec, stream));
          return;
        }
      // capture pays off when keys repeat (the sampler loop: 2 keys); if 32 captures saw fewer hits than captures the caller
      // hands fresh buffers to every call (e.g. a Python loop that keeps every x_{t-1}): replay the launches on the stream
      const bool thrash = pl->graph_captures >= 32 && pl->graph_hits < pl->graph_captures;
      if (thrash) {
        pl->run(stream, nullptr, cache_branch);
        return;
      }
      ++pl->graph_captures;
      if (cap_stream_ == nullptr) IVID_CHECK_CUDA(cudaStreamCreateWithFlags(&cap_stream_, cudaStreamNonBlocking));
      cudaGraph_t graph = nullptr;
      IVID_CHECK_CUDA(cudaStreamBeginCapture(cap_stream_, cudaStreamCaptureModeRelaxed));
      try {
        pl->run(cap_stream_, nullptr, cache_branch);
      } catch (...) {
        cudaStreamEndCapture(cap_stream_, &graph);
        if (graph) cudaGraphDestroy(graph);
        throw;
      }
      IVID_CHECK_CUDA(cudaStreamEndCapture(cap_stream_, &graph));
      cudaGraphExec_t exec = nullptr;
      const cudaError_t ie = cudaGraphInstantiate(&exec, graph, 0);
      cudaGraphDestroy(graph);
      IVID_CHECK_CUDA(ie);
      if (pl->graphs.size() >= 16) {
        // evict the least recently used graph; it may still be executing on the caller's stream
        size_t victim = 0;
        for (size_t i = 1; i < pl->graphs.size(); ++i) if (pl->graphs[i].last_use < pl->graphs[victim].last_use) victim = i;
        IVID_CHECK_CUDA(cudaStreamSynchronize(stream));
        cudaGraphExecDestroy(pl->graphs[victim].exec);
        pl->graphs.erase(pl->graphs.begin() + victim);
      }
      pl->graphs.push_back(Plan::GraphEntry{key, exec, pl->runs});
      IVID_CHECK_CUDA(cudaGraphLaunch(exec, stream));
      return;
    }
    pl->run(stream, nullptr, cache_branch);
    return;
  }
  // profiling pass: every launch bracketed by CUDA events on the launching stream (serialised; shares, not absolutes)
  std::vector<cudaEvent_t> ev(pl->ops.size() + 1);
  for (auto& e : ev) IVID_CHECK_CUDA(cudaEventCreate(&e));
  pl->run(stream, ev.data(), cache_branch);
  IVID_CHECK_CUDA(cudaStreamSynchronize(stream));
  for (size_t i = 0; i < pl->ops.size(); ++i) {
    const Plan::OpRec& op = pl->ops[i];
    if (!pl->kept(op.block, cache_branch)) continue;
    float ms = 0.f;
    IVID_CHECK_CUDA(cudaEventElapsedTime(&ms, ev[i], ev[i + 1]));
    auto& agg = profile_acc_[op.label];
    agg.launches += 1; agg.ms += ms; agg.flops += op.flops; agg.bytes += op.bytes;
    if (!op.note.empty()) {
      char buf[256];
      snprintf(buf, sizeof(buf), "[\"%s\", \"%s\", %.5f, %.4e, %.4e]", op.label, op.note.c_str(), ms, op.flops, op.bytes);
      if (!profile_ops_.empty()) profile_ops_ += ", ";
      profile_ops_ += buf;
    }
  }
  for (auto& e : ev) cudaEventDestroy(e);
}

// Debug tap: output of the named layer (reference module path, e.g. "input_blocks.3.0") of the LAST forward of batch N
// (whatever its input size), converted to fp32 NCHW on the host.  Tensors that only exist as fp16 in the plan (outputs
// nobody reads in fp32) are widened.  Synchronises the device; not on any hot path.
void Unet::debug_tap(int N, const std::string& name, float* host_out, size_t capacity, int* C, int* H, int* W) {
  Plan* pl = nullptr;
  for (auto& p : plans_)
    if (p->N == N && (pl == nullptr || p->last_use > pl->last_use)) pl = p.get();
  if (pl == nullptr) throw Error(kErrState, "debug_tap: no forward of this batch size has run");
  for (const auto& t : pl->taps) {
    if (t.name != name) continue;
    const size_t n = static_cast<size_t>(N) * t.C * t.H * t.W;
    if (C) *C = t.C; if (H) *H = t.H; if (W) *W = t.W;
    if (host_out == nullptr) return;
    IVID_REQUIRE(capacity >= n, "debug_tap: output buffer too small");
    IVID_CHECK_CUDA(cudaSetDevice(device_));
    IVID_CHECK_CUDA(cudaDeviceSynchronize());
    std::vector<float> nhwc(n);
    if (t.d32 != nullptr) {
      IVID_CHECK_CUDA(cudaMemcpy(nhwc.data(), t.d32, n * 4, cudaMemcpyDeviceToHost));
    } else {
      std::vector<__half> h(n);
      IVID_CHECK_CUDA(cudaMemcpy(h.data(), t.d16, n * 2, cudaMemcpyDeviceToHost));
      for (size_t i = 0; i < n; ++i) nhwc[i] = __half2float(h[i]);
    }
    const size_t HW = static_cast<size_t>(t.H) * t.W;
    for (int b = 0; b < N; ++b)
      for (size_t px = 0; px < HW; ++px)
        for (int c = 0; c < t.C; ++c) host_out[(static_cast<size_t>(b) * t.C + c) * HW + px] = nhwc[(static_cast<size_t>(b) * HW + px) * t.C + c];
    return;
  }
  throw Error(kErrInvalidArgument, "debug_tap: unknown layer '" + name + "'");
}

void Unet::profile_begin() { profile_ = true; profile_acc_.clear(); profile_ops_.clear(); }
std::string Unet::profile_end() {
  profile_ = false;
  std::string js = "{";
  bool first = true;
  for (const auto& kv : profile_acc_) {
    if (!first) js += ", ";
    first = false;
    char buf[256];
    snprintf(buf, sizeof(buf), "\"%s\": {\"launches\": %d, \"ms\": %.6f, \"flops\": %.6e, \"bytes\": %.6e}", kv.first.c_str(),
             kv.second.launches, kv.second.ms, kv.second.flops, kv.second.bytes);
    js += buf;
  }
  if (getenv("IVID_PROFILE_OPS") != nullptr) js += ", \"_ops\": [" + profile_ops_ + "]";
  js += "}";
  return js;
}

}  // namespace ivid
