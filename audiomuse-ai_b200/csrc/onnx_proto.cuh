// ONNX ModelProto reader shared by the audio lowering (onnx_model.cu) and the text lowering (text_model.cu):
// protobuf wire format read by hand (there is no protobuf / onnx dependency), initializers converted to fp32 or int64,
// tensor data inline or in an external-data file next to the model (`<name>.onnx.data`, clap_analyzer.py:132-147).
// Above the reader, GraphIndex answers both lowerers' questions about a graph (constants, attributes, consumers, constant
// linears) and finds the LayerNorm, exact-GELU and L2-normalise subgraphs in every form either exporter writes.
#pragma once

#include "common.cuh"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <map>
#include <memory>
#include <set>
#include <string>
#include <vector>

namespace am {
namespace {

// ------------------------------------------------------------------------------------------- protobuf
struct Pb {
  const uint8_t* p;
  const uint8_t* end;
  bool ok = true;
  Pb(const void* d, size_t n) : p((const uint8_t*)d), end((const uint8_t*)d + n) {}
  bool more() const { return ok && p < end; }
  uint64_t varint() {
    uint64_t r = 0;
    for (int s = 0; s < 64; s += 7) {
      if (p >= end) {
        ok = false;
        return 0;
      }
      const uint8_t c = *p++;
      r |= (uint64_t)(c & 0x7f) << s;
      if (!(c & 0x80)) return r;
    }
    ok = false;
    return 0;
  }
  // one field: number, wire type; value in `v` (varint / fixed) or [sub, sub + len)
  bool field(uint32_t* fn, uint32_t* wt, uint64_t* v, const uint8_t** sub, size_t* len) {
    const uint64_t key = varint();
    if (!ok) return false;
    *fn = (uint32_t)(key >> 3);
    *wt = (uint32_t)(key & 7);
    *v = 0;
    *sub = nullptr;
    *len = 0;
    switch (*wt) {
      case 0:
        *v = varint();
        return ok;
      case 1:
        if (end - p < 8) return ok = false;
        std::memcpy(v, p, 8);
        p += 8;
        return true;
      case 5:
        if (end - p < 4) return ok = false;
        std::memcpy(v, p, 4);
        p += 4;
        return true;
      case 2: {
        const uint64_t n = varint();
        if (!ok || n > (uint64_t)(end - p)) return ok = false;
        *sub = p;
        *len = (size_t)n;
        p += n;
        return true;
      }
      default:
        return ok = false;
    }
  }
};

static void packed_ints(uint32_t wt, uint64_t v, const uint8_t* sub, size_t len, std::vector<int64_t>* out) {
  if (wt == 0) {
    out->push_back((int64_t)v);
    return;
  }
  Pb q(sub, len);
  while (q.more()) {
    const uint64_t x = q.varint();
    if (q.ok) out->push_back((int64_t)x);
  }
}
static void packed_floats(uint32_t wt, uint64_t v, const uint8_t* sub, size_t len, std::vector<float>* out) {
  if (wt == 5) {
    float f;
    const uint32_t u = (uint32_t)v;
    std::memcpy(&f, &u, 4);
    out->push_back(f);
    return;
  }
  for (size_t i = 0; i + 4 <= len; i += 4) {
    float f;
    std::memcpy(&f, sub + i, 4);
    out->push_back(f);
  }
}

static float half_to_float(uint16_t h) {
  const uint32_t s = (h >> 15) & 1u, e = (h >> 10) & 31u, m = h & 1023u;
  float v;
  if (e == 0) v = std::ldexp((float)m, -24);
  else if (e == 31) v = m ? NAN : INFINITY;
  else v = std::ldexp((float)(m | 1024u), (int)e - 25);
  return s ? -v : v;
}

struct OTensor {
  std::vector<int64_t> dims;
  int dtype = 1;
  bool is_int = false;
  std::vector<float> f;    // float-typed payloads, converted to fp32
  std::vector<int64_t> i;  // integer-typed payloads
  size_t count() const { return is_int ? i.size() : f.size(); }
  double at(size_t k) const { return is_int ? (double)i[k] : (double)f[k]; }
};

struct OAttr {
  bool has_f = false, has_i = false, has_t = false;
  float f = 0.f;
  int64_t i = 0;
  std::string s;
  OTensor t;
  std::vector<float> floats;
  std::vector<int64_t> ints;
};

struct ONode {
  std::string op, name;
  std::vector<std::string> in, out;
  std::map<std::string, OAttr> attrs;
  bool done = false;
};

struct OGraph {
  std::vector<ONode> nodes;
  std::map<std::string, OTensor> init;
  std::vector<std::string> inputs, outputs;
  int64_t ir_version = 0, opset = 0;
};

static std::string dir_of(const char* path) {
  if (!path) return std::string();
  std::string s(path);
  const size_t k = s.find_last_of('/');
  return k == std::string::npos ? std::string(".") : s.substr(0, k);
}

static int parse_tensor(const uint8_t* d, size_t n, const std::string& base_dir, std::string* name, OTensor* t) {
  Pb pb(d, n);
  uint32_t fn, wt;
  uint64_t v;
  const uint8_t* sub;
  size_t len;
  const uint8_t* raw = nullptr;
  size_t raw_len = 0;
  std::vector<float> f32;
  std::vector<int64_t> i32, i64;
  std::vector<double> f64;
  std::map<std::string, std::string> ext;
  int64_t location = 0;
  while (pb.more() && pb.field(&fn, &wt, &v, &sub, &len)) {
    switch (fn) {
      case 1: packed_ints(wt, v, sub, len, &t->dims); break;
      case 2: t->dtype = (int)v; break;
      case 4: packed_floats(wt, v, sub, len, &f32); break;
      case 5: packed_ints(wt, v, sub, len, &i32); break;
      case 7: packed_ints(wt, v, sub, len, &i64); break;
      case 8: name->assign((const char*)sub, len); break;
      case 9: raw = sub; raw_len = len; break;
      case 10:
        if (wt == 1) {
          double x;
          std::memcpy(&x, &v, 8);
          f64.push_back(x);
        } else {
          for (size_t k = 0; k + 8 <= len; k += 8) {
            double x;
            std::memcpy(&x, sub + k, 8);
            f64.push_back(x);
          }
        }
        break;
      case 13: {
        Pb kv(sub, len);
        std::string key, val;
        uint32_t f2, w2;
        uint64_t v2;
        const uint8_t* s2;
        size_t l2;
        while (kv.more() && kv.field(&f2, &w2, &v2, &s2, &l2)) {
          if (f2 == 1) key.assign((const char*)s2, l2);
          if (f2 == 2) val.assign((const char*)s2, l2);
        }
        ext[key] = val;
        break;
      }
      case 14: location = (int64_t)v; break;
      default: break;
    }
  }
  if (!pb.ok) {
    set_error("onnx: malformed TensorProto");
    return AM_ERR_IO;
  }
  std::vector<uint8_t> ext_buf;
  if (location == 1 || !ext.empty()) {  // external data (model.onnx.data next to the model, clap_analyzer.py:132-147)
    if (base_dir.empty() || !ext.count("location")) {
      set_error("onnx: tensor %s uses external data but the model was given without a path", name->c_str());
      return AM_ERR_IO;
    }
    const std::string fp = base_dir + "/" + ext["location"];
    FILE* f = std::fopen(fp.c_str(), "rb");
    if (!f) {
      set_error("onnx: cannot open external data file %s (tensor %s)", fp.c_str(), name->c_str());
      return AM_ERR_IO;
    }
    const long long off = ext.count("offset") ? std::atoll(ext["offset"].c_str()) : 0;
    long long length = ext.count("length") ? std::atoll(ext["length"].c_str()) : -1;
    if (length < 0) {
      std::fseek(f, 0, SEEK_END);
      length = std::ftell(f) - off;
    }
    ext_buf.resize((size_t)std::max<long long>(length, 0));
    std::fseek(f, (long)off, SEEK_SET);
    const size_t got = ext_buf.empty() ? 0 : std::fread(ext_buf.data(), 1, ext_buf.size(), f);
    std::fclose(f);
    if (got != ext_buf.size()) {
      set_error("onnx: short read of external data for tensor %s", name->c_str());
      return AM_ERR_IO;
    }
    raw = ext_buf.data();
    raw_len = ext_buf.size();
  }
  size_t count = 1;
  for (int64_t x : t->dims) count *= (size_t)std::max<int64_t>(x, 0);
  switch (t->dtype) {
    case 1:  // float
      if (raw) {
        t->f.resize(raw_len / 4);
        std::memcpy(t->f.data(), raw, t->f.size() * 4);
      } else {
        t->f = f32;
      }
      break;
    case 10:  // float16 (raw, or int32_data holding the bit patterns)
      if (raw) {
        t->f.resize(raw_len / 2);
        for (size_t k = 0; k < t->f.size(); ++k) {
          uint16_t h;
          std::memcpy(&h, raw + 2 * k, 2);
          t->f[k] = half_to_float(h);
        }
      } else {
        for (int64_t h : i32) t->f.push_back(half_to_float((uint16_t)h));
      }
      break;
    case 11:  // double
      if (raw) {
        t->f.resize(raw_len / 8);
        for (size_t k = 0; k < t->f.size(); ++k) {
          double x;
          std::memcpy(&x, raw + 8 * k, 8);
          t->f[k] = (float)x;
        }
      } else {
        for (double x : f64) t->f.push_back((float)x);
      }
      break;
    case 7:  // int64
      t->is_int = true;
      if (raw) {
        t->i.resize(raw_len / 8);
        std::memcpy(t->i.data(), raw, t->i.size() * 8);
      } else {
        t->i = i64;
      }
      break;
    case 6:  // int32
      t->is_int = true;
      if (raw) {
        t->i.resize(raw_len / 4);
        for (size_t k = 0; k < t->i.size(); ++k) {
          int32_t x;
          std::memcpy(&x, raw + 4 * k, 4);
          t->i[k] = x;
        }
      } else {
        t->i = i32;
      }
      break;
    case 9:  // bool
      t->is_int = true;
      if (raw) for (size_t k = 0; k < raw_len; ++k) t->i.push_back(raw[k]);
      else t->i = i32;
      break;
    default:
      set_error("onnx: tensor %s has unsupported data_type %d", name->c_str(), t->dtype);
      return AM_ERR_INVALID;
  }
  if (t->count() != count) {
    set_error("onnx: tensor %s holds %zu elements, its dims say %zu", name->c_str(), t->count(), count);
    return AM_ERR_IO;
  }
  return AM_OK;
}

static int parse_attr(const uint8_t* d, size_t n, const std::string& base_dir, std::string* name, OAttr* a) {
  Pb pb(d, n);
  uint32_t fn, wt;
  uint64_t v;
  const uint8_t* sub;
  size_t len;
  while (pb.more() && pb.field(&fn, &wt, &v, &sub, &len)) {
    switch (fn) {
      case 1: name->assign((const char*)sub, len); break;
      case 2: {
        const uint32_t u = (uint32_t)v;
        std::memcpy(&a->f, &u, 4);
        a->has_f = true;
        break;
      }
      case 3: a->i = (int64_t)v; a->has_i = true; break;
      case 4: a->s.assign((const char*)sub, len); break;
      case 5: {
        std::string tn;
        AM_TRY(parse_tensor(sub, len, base_dir, &tn, &a->t));
        a->has_t = true;
        break;
      }
      case 7: packed_floats(wt, v, sub, len, &a->floats); break;
      case 8: packed_ints(wt, v, sub, len, &a->ints); break;
      default: break;
    }
  }
  if (!pb.ok) {
    set_error("onnx: malformed AttributeProto");
    return AM_ERR_IO;
  }
  return AM_OK;
}

static int parse_node(const uint8_t* d, size_t n, const std::string& base_dir, ONode* node) {
  Pb pb(d, n);
  uint32_t fn, wt;
  uint64_t v;
  const uint8_t* sub;
  size_t len;
  while (pb.more() && pb.field(&fn, &wt, &v, &sub, &len)) {
    switch (fn) {
      case 1: node->in.emplace_back((const char*)sub, len); break;
      case 2: node->out.emplace_back((const char*)sub, len); break;
      case 3: node->name.assign((const char*)sub, len); break;
      case 4: node->op.assign((const char*)sub, len); break;
      case 5: {
        std::string an;
        OAttr a;
        AM_TRY(parse_attr(sub, len, base_dir, &an, &a));
        node->attrs[an] = std::move(a);
        break;
      }
      default: break;
    }
  }
  if (!pb.ok) {
    set_error("onnx: malformed NodeProto");
    return AM_ERR_IO;
  }
  return AM_OK;
}

static std::string value_info_name(const uint8_t* d, size_t n) {
  Pb pb(d, n);
  uint32_t fn, wt;
  uint64_t v;
  const uint8_t* sub;
  size_t len;
  while (pb.more() && pb.field(&fn, &wt, &v, &sub, &len))
    if (fn == 1) return std::string((const char*)sub, len);
  return std::string();
}

static int parse_model(const void* data, size_t nbytes, const std::string& base_dir, OGraph* g) {
  Pb pb(data, nbytes);
  uint32_t fn, wt;
  uint64_t v;
  const uint8_t* sub;
  size_t len;
  bool saw_graph = false;
  while (pb.more() && pb.field(&fn, &wt, &v, &sub, &len)) {
    if (fn == 1 && wt == 0) g->ir_version = (int64_t)v;
    if (fn == 8 && wt == 2) {  // opset_import
      Pb q(sub, len);
      uint32_t f2, w2;
      uint64_t v2;
      const uint8_t* s2;
      size_t l2;
      std::string domain;
      int64_t ver = 0;
      while (q.more() && q.field(&f2, &w2, &v2, &s2, &l2)) {
        if (f2 == 1) domain.assign((const char*)s2, l2);
        if (f2 == 2) ver = (int64_t)v2;
      }
      if (domain.empty() || domain == "ai.onnx") g->opset = std::max(g->opset, ver);
    }
    if (fn == 7 && wt == 2) {  // graph
      saw_graph = true;
      Pb q(sub, len);
      uint32_t f2, w2;
      uint64_t v2;
      const uint8_t* s2;
      size_t l2;
      while (q.more() && q.field(&f2, &w2, &v2, &s2, &l2)) {
        if (f2 == 1) {
          ONode node;
          AM_TRY(parse_node(s2, l2, base_dir, &node));
          g->nodes.push_back(std::move(node));
        } else if (f2 == 5) {
          std::string tn;
          OTensor t;
          AM_TRY(parse_tensor(s2, l2, base_dir, &tn, &t));
          g->init[tn] = std::move(t);
        } else if (f2 == 11) {
          g->inputs.push_back(value_info_name(s2, l2));
        } else if (f2 == 12) {
          g->outputs.push_back(value_info_name(s2, l2));
        }
      }
      if (!q.ok) {
        set_error("onnx: malformed GraphProto");
        return AM_ERR_IO;
      }
    }
  }
  if (!pb.ok || !saw_graph || g->nodes.empty()) {
    set_error("onnx: not a ModelProto with a graph (parse %s, %zu nodes)", pb.ok ? "ok" : "failed", g->nodes.size());
    return AM_ERR_IO;
  }
  std::vector<std::string> real_inputs;
  for (const auto& s : g->inputs)
    if (!g->init.count(s)) real_inputs.push_back(s);
  g->inputs = real_inputs;
  return AM_OK;
}

// ------------------------------------------------------------------------------------------- graph queries
// Fails the lowering: am_last_error() names the node (its first output when it has no name) and its operator.
#define LOWER_FAIL(node, ...)                                                                                   \
  do {                                                                                                          \
    char _b[512];                                                                                               \
    std::snprintf(_b, sizeof _b, __VA_ARGS__);                                                                  \
    set_error("onnx: cannot lower node '%s' (%s): %s",                                                          \
              !(node).name.empty() ? (node).name.c_str() : (node).out.empty() ? "" : (node).out[0].c_str(),     \
              (node).op.c_str(), _b);                                                                           \
    return AM_ERR_INVALID;                                                                                      \
  } while (0)

static int64_t attr_i(const ONode& n, const char* k, int64_t dflt) {
  auto it = n.attrs.find(k);
  return it != n.attrs.end() && it->second.has_i ? it->second.i : dflt;
}
static float attr_f(const ONode& n, const char* k, float dflt) {
  auto it = n.attrs.find(k);
  return it != n.attrs.end() && it->second.has_f ? it->second.f : dflt;
}
static std::vector<int64_t> attr_ints(const ONode& n, const char* k) {
  auto it = n.attrs.find(k);
  return it != n.attrs.end() ? it->second.ints : std::vector<int64_t>();
}

static bool close_to(double a, double b, double tol = 1e-5) { return std::fabs(a - b) <= tol * std::max(1.0, std::fabs(b)); }

// A subgraph that both lowerers turn into one operation, whatever form the exporter wrote it in:
//   kLayerNorm  LayerNormalization, or ReduceMean -> Sub -> (Pow 2 | Mul(d, d)) -> ReduceMean -> Add eps -> Sqrt -> Div,
//               then an optional Mul gamma and an optional Add beta
//   kGelu       Gelu (approximate "none"), or x / sqrt 2 | x * sqrt 1/2 -> Erf -> Add 1 -> Mul, with the 0.5 applied to
//               x before that Mul or to its product
//   kL2Norm     ReduceL2 -> [Clip min | Max] -> [Expand] -> Div(x, .)   (F.normalize)
struct Match {
  enum Kind { kLayerNorm, kGelu, kL2Norm } kind = kLayerNorm;
  std::string in, out;     // the value it reads, the value it writes
  std::vector<int> nodes;  // its node indices in graph order: nodes[0] is where a lowerer meets it
  int64_t axis = -1;       // kLayerNorm / kL2Norm: the normalised axis as the graph writes it
  float eps = 0.f;         // kLayerNorm: eps; kL2Norm: the clamp (0 without one)
  bool clamp = false;      // kL2Norm: the norm is clamped from below
  const OTensor *gamma = nullptr, *beta = nullptr;  // kLayerNorm affine (null: 1 and 0)
};

// The queries both lowerers make of one graph: constants (initializers and Constant nodes), who reads and writes each
// value, the graph outputs, and the Match of every LayerNorm, exact GELU and L2-normalise subgraph.
struct GraphIndex {
  OGraph& g;
  std::map<std::string, const OTensor*> consts;
  std::vector<std::unique_ptr<OTensor>> owned;        // value_float / value_int constants
  std::map<std::string, std::vector<int>> consumers;  // a node appears once per input it reads the value on
  std::map<std::string, int> producer;
  std::set<std::string> outputs;
  std::vector<Match> matches;
  std::vector<int> match_at;  // node -> the match it is the first node of, or -1

  explicit GraphIndex(OGraph& g_) : g(g_) {}

  int build() {
    for (auto& kv : g.init) consts[kv.first] = &kv.second;
    for (const auto& o : g.outputs) outputs.insert(o);
    for (size_t i = 0; i < g.nodes.size(); ++i) {
      const ONode& n = g.nodes[i];
      for (const auto& in : n.in)
        if (!in.empty()) consumers[in].push_back((int)i);
      for (const auto& o : n.out) producer[o] = (int)i;
      if (n.op != "Constant" || n.out.empty()) continue;
      auto it = n.attrs.find("value");
      if (it != n.attrs.end() && it->second.has_t) {
        consts[n.out[0]] = &it->second.t;
        continue;
      }
      auto fi = n.attrs.find("value_float");
      auto ii = n.attrs.find("value_int");
      auto t = std::make_unique<OTensor>();
      if (fi != n.attrs.end() && fi->second.has_f) t->f.push_back(fi->second.f);
      else if (ii != n.attrs.end() && ii->second.has_i) {
        t->is_int = true;
        t->i.push_back(ii->second.i);
      } else LOWER_FAIL(n, "Constant without a tensor value");
      consts[n.out[0]] = t.get();
      owned.push_back(std::move(t));
    }
    // every match, so that a lowerer meeting its first node (which may not be the anchor) lowers all of it
    match_at.assign(g.nodes.size(), -1);
    for (size_t i = 0; i < g.nodes.size(); ++i) {
      Match m;
      if (g.nodes[i].in.empty() || g.nodes[i].out.empty() || !(match_layernorm((int)i, &m) || match_gelu((int)i, &m) ||
                                                              match_l2((int)i, &m)))
        continue;
      std::sort(m.nodes.begin(), m.nodes.end());
      match_at[(size_t)m.nodes[0]] = (int)matches.size();
      matches.push_back(std::move(m));
    }
    return AM_OK;
  }

  const OTensor* cst(const std::string& name) const {
    auto it = consts.find(name);
    return it == consts.end() ? nullptr : it->second;
  }
  const OTensor* cin(const ONode& n, size_t idx) const { return idx < n.in.size() && !n.in[idx].empty() ? cst(n.in[idx]) : nullptr; }
  // the single consumer of a value (or -1 when it has several / is a graph output)
  int sole_consumer(const std::string& name) const {
    auto it = consumers.find(name);
    if (it == consumers.end() || it->second.size() != 1 || outputs.count(name)) return -1;
    return it->second[0];
  }
  // integer list given as attribute `k` (older opsets / torch's serializer) or as constant input `idx`
  bool ints_of(const ONode& n, const char* k, size_t idx, std::vector<int64_t>* out) const {
    if (const OTensor* t = cin(n, idx)) {
      out->clear();
      for (size_t q = 0; q < t->count(); ++q) out->push_back((int64_t)t->at(q));
      return true;
    }
    auto it = n.attrs.find(k);
    if (it == n.attrs.end()) return false;
    *out = it->second.ints;
    return true;
  }
  // a one-element constant input `idx`, or float attribute `k` when given
  bool scalar_of(const ONode& n, size_t idx, double* out, const char* k = nullptr) const {
    if (const OTensor* t = cin(n, idx)) {
      if (t->count() != 1) return false;
      *out = t->at(0);
      return true;
    }
    if (!k) return false;
    auto it = n.attrs.find(k);
    if (it == n.attrs.end() || !it->second.has_f) return false;
    *out = it->second.f;
    return true;
  }
  const Match* match_starting(size_t node) const { return match_at[node] < 0 ? nullptr : &matches[(size_t)match_at[node]]; }

  // the constant weight of a MatMul (x @ W, W [K, N]) or a Gemm (W [N, K] under transB) as a row-major [N, K] matrix
  int linear_weight(const ONode& n, int* K, int* N, std::vector<float>* w) const {
    const bool gemm = n.op == "Gemm", tb = gemm && attr_i(n, "transB", 0) != 0;
    if (gemm && (attr_i(n, "transA", 0) != 0 || attr_f(n, "alpha", 1.f) != 1.f || attr_f(n, "beta", 1.f) != 1.f))
      LOWER_FAIL(n, "Gemm with transA / alpha / beta");
    const OTensor* t = cin(n, 1);
    if (!t || t->is_int || t->dims.size() != 2) LOWER_FAIL(n, "weight is not a constant float matrix");
    *K = (int)(tb ? t->dims[1] : t->dims[0]);
    *N = (int)(tb ? t->dims[0] : t->dims[1]);
    w->resize((size_t)*N * *K);
    for (int o = 0; o < *N; ++o)
      for (int k = 0; k < *K; ++k) (*w)[(size_t)o * *K + k] = tb ? t->f[(size_t)o * *K + k] : t->f[(size_t)k * *N + o];
    return AM_OK;
  }

  // ---- matcher helpers
  // v's sole consumer when it has an output and is an `op` (any operator when op is null)
  int reader(const std::string& v, const char* op = nullptr) const {
    const int c = sole_consumer(v);
    return c >= 0 && (!op || g.nodes[c].op == op) && !g.nodes[c].out.empty() ? c : -1;
  }
  int writer(const std::string& v, const char* op) const {
    auto it = producer.find(v);
    return it != producer.end() && g.nodes[it->second].op == op ? it->second : -1;
  }
  // the constant operand of a two-input node whose other input is not constant; *x = that other input
  const OTensor* operand(const ONode& n, std::string* x) const {
    if (n.in.size() != 2) return nullptr;
    for (size_t k = 0; k < 2; ++k)
      if (const OTensor* t = cin(n, k)) {
        if (cin(n, 1 - k)) return nullptr;
        *x = n.in[1 - k];
        return t;
      }
    return nullptr;
  }
  bool scalar_operand(const ONode& n, double want, double tol, std::string* x) const {
    const OTensor* t = operand(n, x);
    return t && t->count() == 1 && close_to(t->at(0), want, tol);
  }
  // a reduction over one axis that keeps it
  bool one_axis(const ONode& n, int64_t* axis) const {
    std::vector<int64_t> ax;
    if (!ints_of(n, "axes", 1, &ax) || ax.size() != 1 || attr_i(n, "keepdims", 1) == 0) return false;
    *axis = ax[0];
    return true;
  }

  // anchored on LayerNormalization, or on the decomposed form's second ReduceMean
  bool match_layernorm(int i, Match* m) const {
    const ONode& n = g.nodes[(size_t)i];
    m->kind = Match::kLayerNorm;
    if (n.op == "LayerNormalization") {
      const OTensor* ga = cin(n, 1);
      if (!ga || ga->is_int) return false;
      m->in = n.in[0];
      m->out = n.out[0];
      m->nodes = {i};
      m->axis = attr_i(n, "axis", -1);
      m->eps = attr_f(n, "epsilon", 1e-5f);
      m->gamma = ga;
      m->beta = cin(n, 2);
      return !m->beta || !m->beta->is_int;
    }
    std::string d, o;
    int64_t axis, axis0;
    if (n.op != "ReduceMean" || !one_axis(n, &axis)) return false;
    const int sq = producer.count(n.in[0]) ? producer.at(n.in[0]) : -1;
    if (sq < 0 || sole_consumer(n.in[0]) != i) return false;
    const ONode& s = g.nodes[(size_t)sq];  // d squared
    if (s.op == "Mul" && s.in.size() == 2 && s.in[0] == s.in[1]) d = s.in[0];
    else if (s.op != "Pow" || !scalar_operand(s, 2.0, 1e-5, &d) || d != s.in[0]) return false;
    const int sb = writer(d, "Sub");
    if (sb < 0 || g.nodes[(size_t)sb].in.size() != 2 || outputs.count(d)) return false;
    const ONode& sub = g.nodes[(size_t)sb];
    const int mn = writer(sub.in[1], "ReduceMean");
    if (mn < 0 || g.nodes[(size_t)mn].in.empty() || g.nodes[(size_t)mn].in[0] != sub.in[0] || sole_consumer(sub.in[1]) != sb ||
        !one_axis(g.nodes[(size_t)mn], &axis0) || axis0 != axis)
      return false;
    int dv = -1;  // d feeds the square and the division only
    for (int c : consumers.at(d))
      if (c != sq) {
        if (dv >= 0 || g.nodes[(size_t)c].op != "Div" || g.nodes[(size_t)c].in[0] != d) return false;
        dv = c;
      }
    const int ae = reader(n.out[0], "Add");
    const OTensor* eps = ae >= 0 ? operand(g.nodes[(size_t)ae], &o) : nullptr;
    if (!eps || eps->count() != 1) return false;
    const int sr = reader(g.nodes[(size_t)ae].out[0], "Sqrt");
    if (sr < 0 || dv < 0 || sole_consumer(g.nodes[(size_t)sr].out[0]) != dv) return false;
    m->in = sub.in[0];
    m->out = g.nodes[(size_t)dv].out[0];
    m->nodes = {mn, sb, sq, i, ae, sr, dv};
    m->axis = axis;
    m->eps = (float)eps->at(0);
    // a per-feature gamma, then a per-feature beta (a scalar is left to the lowerer as an ordinary Mul / Add)
    for (const OTensor** aff : {&m->gamma, &m->beta}) {
      const int q = reader(m->out, aff == &m->gamma ? "Mul" : "Add");
      const OTensor* t = q >= 0 ? operand(g.nodes[(size_t)q], &o) : nullptr;
      if (!t || t->is_int || t->count() < 2) break;
      *aff = t;
      m->nodes.push_back(q);
      m->out = g.nodes[(size_t)q].out[0];
    }
    return true;
  }

  // anchored on Gelu, or on the Erf
  bool match_gelu(int i, Match* m) const {
    const ONode& n = g.nodes[(size_t)i];
    m->kind = Match::kGelu;
    if (n.op == "Gelu") {
      auto it = n.attrs.find("approximate");
      if (it != n.attrs.end() && it->second.s != "none") return false;
      m->in = n.in[0];
      m->out = n.out[0];
      m->nodes = {i};
      return true;
    }
    std::string x, o;
    const int sc = n.op == "Erf" && producer.count(n.in[0]) ? producer.at(n.in[0]) : -1;
    if (sc < 0 || sole_consumer(n.in[0]) != i) return false;
    const ONode& s = g.nodes[(size_t)sc];
    if (!(s.op == "Div" && scalar_operand(s, std::sqrt(2.0), 1e-4, &x) && x == s.in[0]) &&
        !(s.op == "Mul" && scalar_operand(s, std::sqrt(0.5), 1e-4, &x)))
      return false;
    const int ad = reader(n.out[0], "Add");
    if (ad < 0 || !scalar_operand(g.nodes[(size_t)ad], 1.0, 1e-5, &o)) return false;
    const int m1 = reader(g.nodes[(size_t)ad].out[0], "Mul");
    if (m1 < 0 || g.nodes[(size_t)m1].in.size() != 2) return false;
    const ONode& mul = g.nodes[(size_t)m1];
    const std::string& y = mul.in[0] == g.nodes[(size_t)ad].out[0] ? mul.in[1] : mul.in[0];
    int half;
    if (y == x) {  // (x * (1 + erf)) * 0.5
      half = reader(mul.out[0], "Mul");
      if (half < 0 || !scalar_operand(g.nodes[(size_t)half], 0.5, 1e-5, &o)) return false;
      m->out = g.nodes[(size_t)half].out[0];
    } else {  // (x * 0.5) * (1 + erf)
      half = writer(y, "Mul");
      if (half < 0 || sole_consumer(y) != m1 || !scalar_operand(g.nodes[(size_t)half], 0.5, 1e-5, &o) || o != x) return false;
      m->out = mul.out[0];
    }
    m->in = x;
    m->nodes = {sc, i, ad, m1, half};
    return true;
  }

  // anchored on the ReduceL2
  bool match_l2(int i, Match* m) const {
    const ONode& n = g.nodes[(size_t)i];
    m->kind = Match::kL2Norm;
    if (n.op != "ReduceL2" || !one_axis(n, &m->axis)) return false;
    m->nodes = {i};
    std::string v = n.out[0], o;
    int at = reader(v);
    if (at >= 0 && (g.nodes[(size_t)at].op == "Clip" || g.nodes[(size_t)at].op == "Max")) {
      const ONode& c = g.nodes[(size_t)at];
      double lo;
      const OTensor* t = c.op == "Max" ? operand(c, &o) : nullptr;
      if (c.op == "Clip" ? !scalar_of(c, 1, &lo, "min") : !t || t->count() != 1) return false;
      m->eps = (float)(c.op == "Clip" ? lo : t->at(0));
      m->clamp = true;
      m->nodes.push_back(at);
      v = c.out[0];
      at = reader(v);
    }
    if (at >= 0 && g.nodes[(size_t)at].op == "Expand") {
      m->nodes.push_back(at);
      v = g.nodes[(size_t)at].out[0];
      at = reader(v);
    }
    if (at < 0 || g.nodes[(size_t)at].op != "Div" || g.nodes[(size_t)at].in.size() != 2 ||
        g.nodes[(size_t)at].in[0] != n.in[0] || g.nodes[(size_t)at].in[1] != v)
      return false;
    m->in = n.in[0];
    m->out = g.nodes[(size_t)at].out[0];
    m->nodes.push_back(at);
    return true;
  }
};

}  // namespace
}  // namespace am
