// The CLAP text tower on the GPU: ONNX lowering of the deployed RoBERTa text model and its forward pass (sm_90a).
//
// The reference embeds a text query with an onnxruntime session over clap_text_model.onnx
// (tasks/clap_analyzer.py:168-240 loads it, :577-628 and :631-687 run it on {'input_ids', 'attention_mask'} int64
// [B, T] -> 'text_embedding' f32[B, 512]).  The file is TextCLAPWrapper (query/pythorch.sh:95-127): a transformers
// RobertaModel, its pooler tanh(dense(h[:, 0])), Linear -> ReLU -> Linear and F.normalize, exported by the TorchScript
// exporter at opset 17 with constant folding.  am_text_load() reads that file with the shared protobuf reader
// (onnx_proto.cuh) and lowers its node list, following the data flow, to a TextProgram:
//
//   Equal / Not / Cast / CumSum / Mul / Add on input_ids           -> RoBERTa position ids (the pad id from the graph)
//   Gather(word), Gather(position), Add(type row | Gather(1-row))  -> embedding sum, then LayerNorm
//   anything computed from attention_mask and shapes only          -> the key mask (key j is masked where mask == 0)
//   MatMul + Add -> Reshape [.., heads, dh] -> Transpose           -> Q, K, V of one layer (fused into one GEMM)
//   MatMul(Q, K^T) -> Div | Mul, or Mul(Q, s) and Mul(K^T, s)      -> scaled scores (eager or SDPA-symbolic form)
//   -> Add(mask) -> Softmax -> MatMul(V) -> Transpose -> Reshape   -> attention
//   MatMul + Add + Add(residual) + LayerNorm (op or decomposed)    -> output projection / FFN down with residual + LN
//   MatMul + Add + Erf-GELU (any operand order)                    -> FFN up
//   Gather(h, 0, axis 1) -> MatMul|Gemm + Add -> Tanh              -> pooler
//   Gemm -> Relu -> Gemm -> ReduceL2 / Clip / Expand / Div          -> text_projection + F.normalize
//
// and rejects every other node with its name and operator in am_last_error().  L, hidden, heads, FFN, vocabulary,
// positions, pad id, LayerNorm eps and the projection widths all come from the graph.
//
// Forward (text_forward), per (B, T) a TextPlan fixed once:
//   embed_ln_kernel        ids -> position ids (a scan of ids != pad), word + position + type rows, LayerNorm
//   linear_kernel          split-bf16 wgmma GEMM through the shared TMA ring (tma_pipeline.cuh):
//                          D = A_hi.W_hi + A_lo.W_hi + A_hi.W_lo, fp32 accumulation.  Weights are split once at load,
//                          activations by whichever kernel writes them.  A 128 x 64 tile per CTA over a slice of K
//                          (one CTA per SM: ~197 KB of shared memory): when the tiles do not fill the SMs (a single
//                          query, M = 77) K is split into as many balanced slices as fit in one wave, so the idle
//                          SMs stream weight slices; large M runs whole K per tile.  Partial sums go to a workspace.
//   row_epilogue_kernel    sums the K slices in fixed order, then bias, GELU / ReLU / tanh, residual, LayerNorm or
//                          L2 normalise, and writes fp32 and / or the split-bf16 operand of the next GEMM
//   attention_kernel       fp32 scores and online softmax, one CTA per (batch, head, 16 queries), T <= 512
// Every reduction has a fixed order, so a (B, T) input gives the same bits on every run.
#include "common.cuh"
#include "gemm_wgmma.cuh"
#include "onnx_proto.cuh"
#include "tma_pipeline.cuh"

#include <algorithm>
#include <cmath>
#include <map>
#include <memory>
#include <mutex>
#include <set>

namespace am {
namespace text {

enum TAct { kNone = 0, kGelu = 1, kRelu = 2, kTanh = 3 };

struct Linear {
  int K = 0, N = 0;
  std::vector<float> w;  // [N, K] (out, in)
  std::vector<float> b;  // [N] or empty
};

struct LN {
  std::vector<float> g, b;
  float eps = 1e-5f;
};

struct Layer {
  Linear qkv;  // [3H, H]: Q rows, K rows, V rows
  Linear o, f1, f2;
  LN ln1, ln2;
  float scale = 0.f;  // score multiplier (1 / sqrt(dh) in both attention forms)
  bool sdpa = false;  // Q and K^T scaled before their MatMul (the SDPA symbolic) rather than the scores after it
  bool mask_where = false;
};

struct Program {
  int H = 0, heads = 0, dh = 0, ffn = 0, vocab = 0, max_pos = 0, pad_id = 0;
  std::vector<float> word, pos, type_row;  // [vocab, H], [max_pos, H], [H]
  LN emb_ln;
  std::vector<Layer> layers;
  Linear pool, p1, p2;
  bool normalize = false;
  int out_dim() const { return p2.N; }
};

}  // namespace text

namespace {

using text::Linear;
using text::LN;
using text::Program;

// ------------------------------------------------------------------------------------------- lowering
enum TKind {
  tUnknown, tShape, tIds, tMask,
  tPosEq, tPosNe, tPosCum, tPosMul, tPos,          // RoBERTa position ids
  tEmb,                                              // embedding sum (word / pos / type rows)
  tHid,                                              // a LayerNorm output: the hidden state
  tLin,                                              // MatMul (+ bias) of a hidden-like value by a constant
  tRes,                                              // tLin + residual hidden: waiting for its LayerNorm
  tHeads, tScores, tProbs, tCtx, tCtxT, tCtxFlat,    // attention
  tGelu,                                             // GELU of the FFN's up projection
  tTok0, tPooled, tP1, tOut                          // pooler, projection, normalise
};

struct TV {
  int kind = tUnknown;
  std::vector<int64_t> known;  // tShape: elements of a 1-D shape vector, INT64_MIN where unknown
  int64_t pad = 0;             // tPos*: the padding id
  bool word = false, posr = false, type = false;  // tEmb
  int lin = -1;                // tLin / tRes / tHeads: index of the linear; tRes: the LayerNorm's input
  int src = -1;                // tLin: what the MatMul read (a TKind: tHid, tCtxFlat, tGelu, tTok0, tPooled, tP1)
  bool has_bias = false;
  int state = 0;               // tHeads: 0 [B,T,nh,dh], 1 [B,nh,T,dh], 2 [B,nh,dh,T]
  int nh = 0, dh = 0;
  double scale = 1.0;          // tHeads / tScores: multiplier so far
  bool scaled_inputs = false;  // tScores: Q / K^T were scaled (SDPA form)
  bool masked = false;
  int q = -1, k = -1, v = -1;  // tScores / tProbs / tCtx*: linears
};

struct TextLowerer : GraphIndex {
  Program& p;
  std::map<std::string, TV> vals;
  std::vector<Linear> lins;
  // the layer being assembled
  text::Layer cur;
  int stage = 0;  // 0: embeddings, 1: after the embedding LN or a layer's last LN, 2: after attention's LN
  int mask_kind = 0;  // 1 arithmetic (Cast/Sub/Mul), 2 masked_fill (Where)

  TextLowerer(OGraph& g_, Program& p_) : GraphIndex(g_), p(p_) {}

  const TV* val(const std::string& n) const {
    auto it = vals.find(n);
    return it == vals.end() ? nullptr : &it->second;
  }
  bool bias_of(const OTensor* t, int lin) {
    if (!t || t->is_int || (int)t->count() != lins[lin].N) return false;
    if (t->dims.size() > 1)
      for (size_t i = 0; i + 1 < t->dims.size(); ++i)
        if (t->dims[i] != 1) return false;
    if (lins[lin].b.empty()) lins[lin].b = t->f;
    else
      for (int i = 0; i < lins[lin].N; ++i) lins[lin].b[i] += t->f[i];
    return true;
  }

  int node(ONode& n);
  int lower_match(const Match& m);
  int finish_ln(const ONode& n, const TV& x, const Match& m);
  int run();
};

static bool is_int64min(int64_t v) { return v == INT64_MIN; }

int TextLowerer::finish_ln(const ONode& n, const TV& x, const Match& m) {
  if (m.axis != -1 && m.axis != 2) LOWER_FAIL(n, "normalises an axis other than the last");
  const size_t w = m.gamma ? m.gamma->count() : (size_t)p.H;
  LN ln{m.gamma ? m.gamma->f : std::vector<float>(w, 1.f), m.beta ? m.beta->f : std::vector<float>(w, 0.f), m.eps};
  if (ln.g.size() != ln.b.size() || (x.kind != tEmb && (int)ln.g.size() != p.H))
    LOWER_FAIL(n, "LayerNorm affine of %zu / %zu for hidden %d", ln.g.size(), ln.b.size(), p.H);
  TV h;
  h.kind = tHid;
  if (x.kind == tEmb) {
    if (stage != 0 || !x.word || !x.posr) LOWER_FAIL(n, "embedding LayerNorm without word and position rows");
    if (p.H == 0) p.H = (int)ln.g.size();
    if ((int)ln.g.size() != p.H) LOWER_FAIL(n, "LayerNorm of %zu on hidden %d", ln.g.size(), p.H);
    if (p.type_row.empty()) p.type_row.assign((size_t)p.H, 0.f);
    p.emb_ln = ln;
    stage = 1;
  } else if (x.kind == tRes) {
    const TV& l = x;  // tRes carries the linear and what it read
    if (l.src == tCtxFlat) {
      if (stage != 1 || cur.qkv.N == 0) LOWER_FAIL(n, "attention output LayerNorm out of order");
      cur.o = lins[l.lin];
      cur.ln1 = ln;
      stage = 2;
    } else if (l.src == tGelu) {
      if (stage != 2 || cur.f1.N == 0) LOWER_FAIL(n, "FFN LayerNorm out of order");
      cur.f2 = lins[l.lin];
      cur.ln2 = ln;
      p.layers.push_back(std::move(cur));
      cur = text::Layer();
      stage = 1;
    } else {
      LOWER_FAIL(n, "residual LayerNorm after an unexpected linear");
    }
  } else {
    LOWER_FAIL(n, "LayerNorm of a value that is neither the embedding sum nor a residual sum");
  }
  vals[m.out] = h;
  return AM_OK;
}

// a LayerNorm, GELU or F.normalize: lowered where the model has one, rejected anywhere else
int TextLowerer::lower_match(const Match& m) {
  const ONode& n = g.nodes[(size_t)m.nodes[0]];
  const TV* x = val(m.in);
  if (!x) LOWER_FAIL(n, "input '%s' is not produced by a supported node", m.in.c_str());
  if (m.kind == Match::kLayerNorm) return finish_ln(n, *x, m);
  if (m.kind == Match::kGelu) {
    if (x->kind != tLin || x->src != tHid || stage != 2) LOWER_FAIL(n, "GELU of a value other than the FFN's up projection");
    TV v = *x;
    v.kind = tGelu;
    vals[m.out] = v;
    return AM_OK;
  }
  if (x->kind != tLin || x->src != tP1) LOWER_FAIL(n, "L2 normalise of a value other than the projection");
  if (m.axis != -1 && m.axis != 1) LOWER_FAIL(n, "norm over an axis other than the last");
  if (!m.clamp || m.eps <= 0 || m.eps > 1e-6) LOWER_FAIL(n, "norm clamp other than F.normalize's");
  p.p2 = lins[x->lin];
  p.normalize = true;
  TV v;
  v.kind = tOut;
  vals[m.out] = v;
  return AM_OK;
}

int TextLowerer::node(ONode& n) {
  const std::string& op = n.op;
  if (n.out.empty()) LOWER_FAIL(n, "no output");
  // inputs: constants, or values with a kind
  std::vector<const TV*> in(n.in.size(), nullptr);
  bool all_const = true, shape_or_const = true, mask_like = true;
  for (size_t i = 0; i < n.in.size(); ++i) {
    if (n.in[i].empty() || cst(n.in[i])) continue;
    all_const = false;
    in[i] = val(n.in[i]);
    if (!in[i]) LOWER_FAIL(n, "input '%s' is not produced by a supported node", n.in[i].c_str());
    if (in[i]->kind != tShape) shape_or_const = false;
    if (in[i]->kind != tShape && in[i]->kind != tMask) mask_like = false;
  }
  auto kind = [&](size_t i) { return i < in.size() && in[i] ? in[i]->kind : -1; };
  auto out = [&](TV v) { vals[n.out[0]] = std::move(v); return AM_OK; };
  static const std::set<std::string> kShapeOps = {"Shape", "Gather", "Unsqueeze", "Squeeze", "Concat", "Reshape",
                                                  "ConstantOfShape", "Mul", "Add", "Sub", "Div", "Equal", "Where",
                                                  "Cast", "Slice", "Range", "Expand", "Not", "Identity"};

  if (all_const && op != "Shape") LOWER_FAIL(n, "operator on constants only (not folded at export)");
  if (op == "Shape") {
    TV v;
    v.kind = tShape;
    return out(v);
  }
  if (shape_or_const) {
    if (!kShapeOps.count(op)) LOWER_FAIL(n, "operator not supported in shape arithmetic");
    TV v;
    v.kind = tShape;
    if (op == "Concat") {
      for (size_t i = 0; i < n.in.size(); ++i) {
        if (const OTensor* t = cst(n.in[i])) {
          for (size_t q = 0; q < t->count(); ++q) v.known.push_back((int64_t)t->at(q));
        } else if (!in[i]->known.empty()) {
          v.known.insert(v.known.end(), in[i]->known.begin(), in[i]->known.end());
        } else {
          v.known.push_back(INT64_MIN);  // an Unsqueeze of a dimension read from a shape
        }
      }
    }
    return out(v);
  }
  if (mask_like && (kind(0) == tMask || kind(1) == tMask || kind(2) == tMask)) {
    static const std::set<std::string> kMaskOps = {"Unsqueeze", "Cast", "Sub", "Mul", "Where", "Expand", "Equal", "Not",
                                                   "Reshape", "Identity", "Slice", "Squeeze"};
    if (!kMaskOps.count(op)) LOWER_FAIL(n, "operator not supported in the attention-mask construction");
    if (op == "Where") mask_kind = 2;
    if (op == "Mul" && mask_kind == 0) mask_kind = 1;
    TV v;
    v.kind = tMask;
    return out(v);
  }
  // mask values built from the mask input directly
  if (op == "Unsqueeze" || op == "Cast" || op == "Expand" || op == "Reshape" || op == "Identity") {
    if (kind(0) == tMask) {
      TV v;
      v.kind = tMask;
      return out(v);
    }
  }
  if (op == "Identity" || op == "Dropout") {
    if (!in[0]) LOWER_FAIL(n, "identity of a constant");
    return out(*in[0]);
  }
  if (op == "Cast") {
    const int k = kind(0);
    if (k == tPosNe || k == tPosMul || k == tPos || k == tPosCum) return out(*in[0]);
    LOWER_FAIL(n, "Cast of an unsupported value");
  }

  // ---------------------------------------------------------------- position ids
  if (op == "Equal" && kind(0) == tIds) {
    double c;
    if (!scalar_of(n, 1, &c)) LOWER_FAIL(n, "input_ids compared with a non-constant");
    TV v;
    v.kind = tPosEq;
    v.pad = (int64_t)c;
    return out(v);
  }
  if (op == "Not" && kind(0) == tPosEq) {
    TV v = *in[0];
    v.kind = tPosNe;
    return out(v);
  }
  if (op == "CumSum" && kind(0) == tPosNe) {
    double ax;
    if (!scalar_of(n, 1, &ax) || (ax != 1 && ax != -1)) LOWER_FAIL(n, "cumulative sum over an axis other than the sequence");
    TV v = *in[0];
    v.kind = tPosCum;
    return out(v);
  }
  if (op == "Mul" && ((kind(0) == tPosCum && kind(1) == tPosNe) || (kind(0) == tPosNe && kind(1) == tPosCum))) {
    TV v = *in[0];
    v.kind = tPosMul;
    return out(v);
  }
  if (op == "Add" && (kind(0) == tPosMul || kind(1) == tPosMul)) {
    double c;
    const TV& a = *(kind(0) == tPosMul ? in[0] : in[1]);
    if (!scalar_of(n, kind(0) == tPosMul ? 1 : 0, &c) || (int64_t)c != a.pad)
      LOWER_FAIL(n, "position ids offset by something other than the padding id %lld", (long long)a.pad);
    TV v = a;
    v.kind = tPos;
    return out(v);
  }

  // ---------------------------------------------------------------- embeddings
  if (op == "Gather") {
    const OTensor* tab = cin(n, 0);
    const int axis = (int)attr_i(n, "axis", 0);
    if (tab && axis == 0 && tab->dims.size() == 2 && !tab->is_int) {
      TV v;
      v.kind = tEmb;
      if (kind(1) == tIds) {
        if (!p.word.empty()) LOWER_FAIL(n, "a second word-embedding gather");
        p.vocab = (int)tab->dims[0];
        p.H = (int)tab->dims[1];
        p.word = tab->f;
        v.word = true;
      } else if (kind(1) == tPos) {
        if (!p.pos.empty()) LOWER_FAIL(n, "a second position-embedding gather");
        if (p.H && tab->dims[1] != p.H) LOWER_FAIL(n, "position table width %lld, hidden %d", (long long)tab->dims[1], p.H);
        p.max_pos = (int)tab->dims[0];
        p.pad_id = (int)in[1]->pad;
        p.pos = tab->f;
        v.posr = true;
      } else if (kind(1) == tShape && tab->dims[0] == 1) {  // token types: a one-row table, so always row 0
        p.type_row = tab->f;
        v.type = true;
      } else {
        LOWER_FAIL(n, "gather from a table by an index that is neither input_ids nor the position ids");
      }
      return out(v);
    }
    if (kind(0) == tHid && axis == 1) {
      double c;
      if (!scalar_of(n, 1, &c) || c != 0) LOWER_FAIL(n, "pooler reads a token other than the first");
      TV v;
      v.kind = tTok0;
      return out(v);
    }
    LOWER_FAIL(n, "unsupported gather");
  }
  if (op == "Add" && (kind(0) == tEmb || kind(1) == tEmb)) {
    TV v;
    v.kind = tEmb;
    for (int i = 0; i < 2; ++i) {
      if (kind(i) == tEmb) {
        v.word |= in[i]->word;
        v.posr |= in[i]->posr;
        v.type |= in[i]->type;
      } else if (const OTensor* t = cin(n, i)) {  // the constant-folded token-type row
        if (p.H == 0 || (int)t->count() != p.H || v.type) LOWER_FAIL(n, "embedding sum plus a constant of %zu values", t->count());
        p.type_row = t->f;
        v.type = true;
      } else {
        LOWER_FAIL(n, "embedding sum plus an unsupported value");
      }
    }
    return out(v);
  }

  // ---------------------------------------------------------------- linears
  if (op == "MatMul" || op == "Gemm") {
    const int k0 = kind(0);
    if (k0 == tHid || k0 == tCtxFlat || k0 == tGelu || k0 == tTok0 || k0 == tPooled || k0 == tP1) {
      if (k0 == tGelu) {  // the FFN's down projection: the linear that fed GELU was its up projection
        if (stage != 2 || cur.f1.N) LOWER_FAIL(n, "FFN out of order");
        cur.f1 = lins[in[0]->lin];
        p.ffn = cur.f1.N;
      }
      const int K = k0 == tGelu ? p.ffn : (k0 == tP1 ? 0 : p.H);
      Linear L;
      AM_TRY(linear_weight(n, &L.K, &L.N, &L.w));
      if (K && L.K != K) LOWER_FAIL(n, "weight must be a constant [%d, N] matrix", K);
      lins.push_back(std::move(L));
      const int li = (int)lins.size() - 1;
      TV v;
      v.kind = tLin;
      v.lin = li;
      v.src = k0;
      if (op == "Gemm" && n.in.size() > 2 && !n.in[2].empty()) {
        if (!bias_of(cin(n, 2), li)) LOWER_FAIL(n, "non-constant or mis-sized bias");
        v.has_bias = true;
      }
      return out(v);
    }
    if (op == "MatMul" && kind(0) == tHeads && kind(1) == tHeads) {
      const TV &q = *in[0], &k = *in[1];
      if (q.state != 1 || k.state != 2) LOWER_FAIL(n, "scores need Q as [B, heads, T, dh] and K as [B, heads, dh, T]");
      TV v;
      v.kind = tScores;
      v.q = q.lin;
      v.k = k.lin;
      v.nh = q.nh;
      v.dh = q.dh;
      v.scale = q.scale * k.scale;
      v.scaled_inputs = q.scale != 1.0 || k.scale != 1.0;
      return out(v);
    }
    if (op == "MatMul" && kind(0) == tProbs && kind(1) == tHeads) {
      if (in[1]->state != 1) LOWER_FAIL(n, "V must be [B, heads, T, dh]");
      TV v = *in[0];
      v.kind = tCtx;
      v.v = in[1]->lin;
      return out(v);
    }
    LOWER_FAIL(n, "matrix product of unsupported operands");
  }
  if (op == "Add" && (kind(0) == tLin || kind(1) == tLin) && (cin(n, 0) || cin(n, 1))) {
    TV v = *in[kind(0) == tLin ? 0 : 1];
    if (v.has_bias) LOWER_FAIL(n, "second bias on a linear");
    if (!bias_of(cin(n, kind(0) == tLin ? 1 : 0), v.lin)) LOWER_FAIL(n, "bias does not match the linear's %d outputs", lins[v.lin].N);
    v.has_bias = true;
    return out(v);
  }
  if (op == "Add" && ((kind(0) == tLin && kind(1) == tHid) || (kind(0) == tHid && kind(1) == tLin))) {
    TV v = *in[kind(0) == tLin ? 0 : 1];
    if (v.src != tCtxFlat && v.src != tGelu) LOWER_FAIL(n, "residual added to an unexpected linear");
    v.kind = tRes;
    return out(v);
  }

  // ---------------------------------------------------------------- attention
  if (op == "Reshape" && kind(0) == tLin) {
    const TV* s = in[1];
    std::vector<int64_t> shp;
    if (const OTensor* t = cin(n, 1)) {
      for (size_t q = 0; q < t->count(); ++q) shp.push_back((int64_t)t->at(q));
    } else if (s && s->kind == tShape) {
      shp = s->known;
    }
    if (shp.size() != 4 || is_int64min(shp[2]) || is_int64min(shp[3])) LOWER_FAIL(n, "split into heads needs a constant [.., heads, dh] tail");
    int64_t nh = shp[2], dh = shp[3];
    const int N = lins[in[0]->lin].N;
    if (nh == -1 && dh > 0) nh = N / dh;
    if (dh == -1 && nh > 0) dh = N / nh;
    if (nh <= 0 || dh <= 0 || nh * dh != N) LOWER_FAIL(n, "%lld heads of %lld for %d features", (long long)nh, (long long)dh, N);
    TV v = *in[0];
    v.kind = tHeads;
    v.state = 0;
    v.nh = (int)nh;
    v.dh = (int)dh;
    return out(v);
  }
  if (op == "Transpose" && (kind(0) == tHeads || kind(0) == tCtx)) {
    const std::vector<int64_t> perm = attr_ints(n, "perm");
    TV v = *in[0];
    if (v.kind == tCtx) {
      if (perm != std::vector<int64_t>{0, 2, 1, 3}) LOWER_FAIL(n, "context transposed other than back to [B, T, heads, dh]");
      v.kind = tCtxT;
      return out(v);
    }
    if (v.state == 0 && perm == std::vector<int64_t>{0, 2, 1, 3}) v.state = 1;
    else if (v.state == 0 && perm == std::vector<int64_t>{0, 2, 3, 1}) v.state = 2;
    else if (v.state == 1 && perm == std::vector<int64_t>{0, 1, 3, 2}) v.state = 2;
    else LOWER_FAIL(n, "unsupported head transpose");
    return out(v);
  }
  if ((op == "Mul" || op == "Div") && (kind(0) == tHeads || kind(0) == tScores)) {
    double c;
    if (!scalar_of(n, 1, &c) || c == 0) LOWER_FAIL(n, "scaled by a non-constant");
    TV v = *in[0];
    if (v.kind == tScores && v.masked) LOWER_FAIL(n, "scale after the mask");
    v.scale *= op == "Mul" ? c : 1.0 / c;
    return out(v);
  }
  if (op == "Add" && ((kind(0) == tScores && kind(1) == tMask) || (kind(0) == tMask && kind(1) == tScores))) {
    TV v = *in[kind(0) == tScores ? 0 : 1];
    if (v.masked) LOWER_FAIL(n, "second mask");
    v.masked = true;
    return out(v);
  }
  if (op == "Softmax" && kind(0) == tScores) {
    const int64_t ax = attr_i(n, "axis", -1);
    if (ax != -1 && ax != 3) LOWER_FAIL(n, "softmax over axis %lld", (long long)ax);
    if (!in[0]->masked) LOWER_FAIL(n, "scores without the attention mask");
    TV v = *in[0];
    v.kind = tProbs;
    return out(v);
  }
  if (op == "Reshape" && kind(0) == tCtxT) {
    TV v = *in[0];
    const int Hh = v.nh * v.dh;
    std::vector<int64_t> shp;
    if (const OTensor* t = cin(n, 1)) for (size_t q = 0; q < t->count(); ++q) shp.push_back((int64_t)t->at(q));
    else if (in[1] && in[1]->kind == tShape) shp = in[1]->known;
    if (shp.size() != 3 || (shp[2] != Hh && shp[2] != -1)) LOWER_FAIL(n, "context not merged back to [B, T, %d]", Hh);
    // the layer's Q, K, V: one fused linear [3H, H]
    if (stage != 1 || cur.qkv.N) LOWER_FAIL(n, "attention out of order");
    const Linear &q = lins[v.q], &k = lins[v.k], &vv = lins[v.v];
    if (q.N != p.H || k.N != p.H || vv.N != p.H) LOWER_FAIL(n, "Q / K / V widths %d / %d / %d for hidden %d", q.N, k.N, vv.N, p.H);
    if (p.heads && (p.heads != v.nh || p.dh != v.dh)) LOWER_FAIL(n, "%d heads of %d after %d of %d", v.nh, v.dh, p.heads, p.dh);
    p.heads = v.nh;
    p.dh = v.dh;
    Linear f;
    f.K = p.H;
    f.N = 3 * p.H;
    for (const Linear* l : {&q, &k, &vv}) {
      f.w.insert(f.w.end(), l->w.begin(), l->w.end());
      if (l->b.empty()) f.b.insert(f.b.end(), (size_t)p.H, 0.f);
      else f.b.insert(f.b.end(), l->b.begin(), l->b.end());
    }
    cur.qkv = std::move(f);
    cur.scale = (float)v.scale;
    cur.sdpa = v.scaled_inputs;
    cur.mask_where = mask_kind == 2;
    v.kind = tCtxFlat;
    return out(v);
  }

  // ---------------------------------------------------------------- pooler, projection, normalise
  if (op == "Tanh" && kind(0) == tLin && in[0]->src == tTok0) {
    if (!in[0]->has_bias) LOWER_FAIL(n, "pooler without a bias");
    p.pool = lins[in[0]->lin];
    TV v;
    v.kind = tPooled;
    return out(v);
  }
  if (op == "Relu" && kind(0) == tLin && in[0]->src == tPooled) {
    p.p1 = lins[in[0]->lin];
    TV v;
    v.kind = tP1;
    return out(v);
  }
  LOWER_FAIL(n, "operator not supported here");
}

int TextLowerer::run() {
  if (g.inputs.size() != 2) {
    set_error("onnx: the text model needs the inputs input_ids and attention_mask (the graph has %zu inputs)", g.inputs.size());
    return AM_ERR_INVALID;
  }
  for (const std::string& s : g.inputs) {
    TV v;
    if (s == "input_ids") v.kind = tIds;
    else if (s == "attention_mask") v.kind = tMask;
    else {
      set_error("onnx: unexpected text-model input '%s' (want input_ids, attention_mask)", s.c_str());
      return AM_ERR_INVALID;
    }
    vals[s] = v;
  }
  AM_TRY(build());
  for (size_t i = 0; i < g.nodes.size(); ++i) {
    ONode& n = g.nodes[i];
    if (n.done || n.op == "Constant") continue;  // Constant nodes are registered by the index
    if (const Match* m = match_starting(i)) {
      AM_TRY(lower_match(*m));
      for (int q : m->nodes) g.nodes[(size_t)q].done = true;
    } else {
      AM_TRY(node(n));
    }
  }
  if (g.outputs.size() != 1 || !val(g.outputs[0]) || val(g.outputs[0])->kind != tOut) {
    set_error("onnx: the graph's output is not an L2-normalised projection of the pooled hidden state");
    return AM_ERR_INVALID;
  }
  if (stage != 1 || p.layers.empty()) {
    set_error("onnx: the graph ends inside a transformer layer (%zu complete layers)", p.layers.size());
    return AM_ERR_INVALID;
  }
  p.ffn = p.layers[0].f1.N;
  for (const auto& L : p.layers)
    if (L.f1.N != p.ffn || L.f1.K != p.H || L.f2.K != p.ffn || L.f2.N != p.H || L.o.K != p.H || L.o.N != p.H) {
      set_error("onnx: layers of different shapes");
      return AM_ERR_INVALID;
    }
  if (p.pool.K != p.H || p.pool.N != p.H || p.p1.K != p.H || p.p2.K != p.p1.N) {
    set_error("onnx: pooler %dx%d / projection %dx%d, %dx%d do not chain from hidden %d", p.pool.N, p.pool.K, p.p1.N,
              p.p1.K, p.p2.N, p.p2.K, p.H);
    return AM_ERR_INVALID;
  }
  if (p.dh > 64) {
    set_error("onnx: head dimension %d (the attention kernel takes up to 64)", p.dh);
    return AM_ERR_INVALID;
  }
  return AM_OK;
}

}  // namespace

// ------------------------------------------------------------------------------------------- kernels
namespace {

using pipe::kChunkK;

constexpr int kTileM = 128;                         // two consumer warpgroups of 64 rows
constexpr int kTileN = 64;                          // weight rows per tile
constexpr int kATile = kTileM * kChunkK * 2;        // 16 KiB: one of A_hi, A_lo
constexpr int kWTile = kTileN * kChunkK * 2;        // 8 KiB: one of W_hi, W_lo
constexpr int kStageBytes = 2 * kATile + 2 * kWTile;  // 48 KiB
constexpr int kStages = 4;
using Ring = pipe::Ring<kStages>;
constexpr size_t kLinearSmem = Ring::smem_bytes(kStageBytes, kStages, 0);

__host__ __device__ inline int kpad(int k) { return (k + 63) / 64 * 64; }

// P[split, M, N] = A[M, K-slice] . W[N, K-slice]^T with A = A_hi + A_lo and W = W_hi + W_lo (each stored [rows, 2 Kp]
// as hi | lo): hi.hi + lo.hi + hi.lo per 16-wide K step, fp32 accumulation.  Grid (N tiles, M tiles, K slices); the
// slice z of the S = gridDim.z slices covers chunks [z num_kb / S, (z + 1) num_kb / S) (S <= num_kb, none empty).
__global__ void __launch_bounds__(pipe::kThreads, 1)
linear_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_w, int M, int N,
              int Kp, float* __restrict__ P) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  Ring ring(smem_raw, kStageBytes, kStages, 0);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_kb = Kp / kChunkK;
  const int kb0 = (int)((int64_t)blockIdx.z * num_kb / gridDim.z), kb1 = (int)((int64_t)(blockIdx.z + 1) * num_kb / gridDim.z);
  const int n0 = blockIdx.x * kTileN, m0 = blockIdx.y * kTileM;
  if (threadIdx.x == 0) {
    ptx::prefetch_tensormap(&map_a);
    ptx::prefetch_tensormap(&map_w);
    ring.init();
  }
  __syncthreads();
  if (warp < 4) {
    ptx::regs_producer();
    if (warp == 0 && ptx::elect_one_sync()) {
      for (int kb = kb0; kb < kb1; ++kb) {
        const Ring::Slot s = ring.acquire();
        ptx::tma_load_2d(s.smem, &map_a, s.bar, kb * kChunkK, m0);
        ptx::tma_load_2d(s.smem + kATile, &map_a, s.bar, Kp + kb * kChunkK, m0);
        ptx::tma_load_2d(s.smem + 2 * kATile, &map_w, s.bar, kb * kChunkK, n0);
        ptx::tma_load_2d(s.smem + 2 * kATile + kWTile, &map_w, s.bar, Kp + kb * kChunkK, n0);
      }
    }
    return;
  }
  ptx::regs_consumer();
  const int wg = (threadIdx.x >> 7) - 1;
  float acc[kTileN / 2];
#pragma unroll
  for (int i = 0; i < kTileN / 2; ++i) acc[i] = 0.f;
  for (int kb = kb0; kb < kb1; ++kb) {
    const uint32_t s = ring.wait();
    const uint32_t rows = (uint32_t)(wg * 64 * 128);
    pipe::mma_chunk_split<kTileN, false>(acc, s + rows, s + kATile + rows, s + 2 * kATile, s + 2 * kATile + kWTile,
                                         kb - kb0);
    ring.release();
  }
  const int quad = lane & 3;
  const int row0 = m0 + wg * 64 + ((threadIdx.x & 127) >> 5) * 16 + (lane >> 2);
  float* out = P + (size_t)blockIdx.z * M * N;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = row0 + 8 * h;
    if (row >= M) continue;
#pragma unroll
    for (int j = 0; j < kTileN / 8; ++j) {
      const int c = n0 + 8 * j + 2 * quad;
      float* o = &out[(size_t)row * N + c];
      if ((N & 1) == 0) {  // c is even: the pair is 8-byte aligned, and c < N means c + 1 < N
        if (c < N) *reinterpret_cast<float2*>(o) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
      } else {  // odd N: one float at a time
        if (c < N) o[0] = acc[4 * j + 2 * h];
        if (c + 1 < N) o[1] = acc[4 * j + 2 * h + 1];
      }
    }
  }
}

struct EpiArgs {
  const float* P = nullptr;  // [splits, M, N]
  int splits = 1, M = 0, N = 0;
  const float* bias = nullptr;      // [N]
  int act = text::kNone;
  const float* residual = nullptr;  // [M, N] added after the activation
  const float* ln_g = nullptr;      // LayerNorm over the row (after the residual)
  const float* ln_b = nullptr;
  float eps = 0.f;
  bool l2 = false;                  // x / max(||x||, 1e-12) over the row
  float* out = nullptr;             // [M, N] fp32
  __nv_bfloat16* out_split = nullptr;  // [M, 2 Np] hi | lo, Np = N rounded up to 64 (zero tail)
};

constexpr int kRowThreads = 256;

// deterministic block sum: warp trees, then the warps' partials in order
__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = 0.f;
  for (int w = 0; w < kRowThreads / 32; ++w) t += red[w];
  return t;
}

__device__ __forceinline__ float act_f(float v, int act) {
  switch (act) {
    case text::kGelu: return 0.5f * v * (1.0f + erff(v * 0.70710678118654752f));
    case text::kRelu: return fmaxf(v, 0.f);
    case text::kTanh: return tanhf(v);
    default: return v;
  }
}

__device__ __forceinline__ void store_split(__nv_bfloat16* row, int Np, int c, float v) {
  const __nv_bfloat16 hi = __float2bfloat16_rn(v);
  row[c] = hi;
  row[Np + c] = __float2bfloat16_rn(v - __bfloat162float(hi));
}

// one CTA per row: the K slices summed in order, bias, activation, residual, LayerNorm / L2, the stores
__global__ void __launch_bounds__(kRowThreads) row_epilogue_kernel(const EpiArgs a) {
  extern __shared__ float xs[];  // [N]
  __shared__ float red[kRowThreads / 32];
  const int m = blockIdx.x;
  const int N = a.N;
  const size_t MN = (size_t)a.M * N;
  float part = 0.f;
  for (int c = threadIdx.x; c < N; c += kRowThreads) {
    const float* p = a.P + (size_t)m * N + c;
    float v = p[0];
    for (int s = 1; s < a.splits; ++s) v += p[s * MN];
    if (a.bias) v += a.bias[c];
    v = act_f(v, a.act);
    if (a.residual) v += a.residual[(size_t)m * N + c];
    xs[c] = v;
    part += v;
  }
  if (a.ln_g) {
    const float mean = block_sum(part, red) / (float)N;
    float q = 0.f;
    for (int c = threadIdx.x; c < N; c += kRowThreads) {
      const float d = xs[c] - mean;
      q = fmaf(d, d, q);
    }
    const float var = block_sum(q, red) / (float)N;
    const float rs = 1.0f / sqrtf(var + a.eps);
    for (int c = threadIdx.x; c < N; c += kRowThreads) xs[c] = (xs[c] - mean) * rs * a.ln_g[c] + a.ln_b[c];
  } else if (a.l2) {
    float q = 0.f;
    for (int c = threadIdx.x; c < N; c += kRowThreads) q = fmaf(xs[c], xs[c], q);
    const float nrm = fmaxf(sqrtf(block_sum(q, red)), 1e-12f);
    for (int c = threadIdx.x; c < N; c += kRowThreads) xs[c] = xs[c] / nrm;
  }
  const int Np = kpad(N);
  for (int c = threadIdx.x; c < Np; c += kRowThreads) {
    const float v = c < N ? xs[c] : 0.f;
    if (a.out && c < N) a.out[(size_t)m * N + c] = v;
    if (a.out_split) store_split(a.out_split + (size_t)m * 2 * Np, Np, c, v);
  }
}

// one CTA per token (b, t): RoBERTa's position id (cumsum of ids != pad up to t, times ids[t] != pad, plus pad),
// word + position + type rows, LayerNorm; writes the hidden state fp32 and split
__global__ void __launch_bounds__(kRowThreads)
embed_ln_kernel(const int64_t* __restrict__ ids, int T, int H, int pad, const float* __restrict__ word,
                const float* __restrict__ pos, const float* __restrict__ type_row, const float* __restrict__ g,
                const float* __restrict__ b, float eps, float* __restrict__ out, __nv_bfloat16* __restrict__ out_split) {
  extern __shared__ float xs[];  // [H]
  __shared__ float red[kRowThreads / 32];
  const int m = blockIdx.x, bt = m / T, t = m % T;
  const int64_t* row = ids + (size_t)bt * T;
  float cnt = 0.f;
  for (int j = threadIdx.x; j <= t; j += kRowThreads) cnt += row[j] != pad ? 1.f : 0.f;
  const int total = (int)block_sum(cnt, red);
  const int64_t id = row[t];
  const int p = id != pad ? total + pad : pad;
  float part = 0.f;
  for (int c = threadIdx.x; c < H; c += kRowThreads) {
    const float v = word[(size_t)id * H + c] + pos[(size_t)p * H + c] + type_row[c];
    xs[c] = v;
    part += v;
  }
  const float mean = block_sum(part, red) / (float)H;
  float q = 0.f;
  for (int c = threadIdx.x; c < H; c += kRowThreads) {
    const float d = xs[c] - mean;
    q = fmaf(d, d, q);
  }
  const float rs = 1.0f / sqrtf(block_sum(q, red) / (float)H + eps);
  const int Hp = kpad(H);
  for (int c = threadIdx.x; c < Hp; c += kRowThreads) {
    const float v = c < H ? (xs[c] - mean) * rs * g[c] + b[c] : 0.f;
    if (c < H) out[(size_t)m * H + c] = v;
    store_split(out_split + (size_t)m * 2 * Hp, Hp, c, v);
  }
}

constexpr int kAttnQ = 16;      // queries per CTA
constexpr int kAttnWarps = 4;   // each warp takes queries warp, warp + 4, ...
constexpr int kAttnKeys = 32;   // keys staged per step (one per lane)

// Masked attention of one (batch, head, 16-query tile): qkv f32 [B T, 3H] (Q | K | V), key j of batch b masked where
// mask[b, j] == 0 (a batch row with no unmasked key attends uniformly, as the additive finfo.min mask does);
// scores s = scale q.k in fp32, online softmax, output written split to ctx [B T, 2 Hp].
__global__ void __launch_bounds__(kAttnWarps * 32)
attention_kernel(const float* __restrict__ qkv, const int64_t* __restrict__ mask, int T, int H, int heads, int dh,
                 float scale, __nv_bfloat16* __restrict__ ctx) {
  __shared__ float qs[kAttnQ][64];
  __shared__ float ks[kAttnKeys][65];
  __shared__ float vs[kAttnKeys][64];
  const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * kAttnQ;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const size_t ld = 3 * (size_t)H;
  const float* base = qkv + (size_t)b * T * ld + (size_t)h * dh;
  const int64_t* mrow = mask + (size_t)b * T;
  // any unmasked key in this batch row?
  int any = 0;
  for (int j = threadIdx.x; j < T; j += blockDim.x) any |= mrow[j] != 0;
  any = __syncthreads_or(any);
  for (int i = threadIdx.x; i < kAttnQ * 64; i += blockDim.x) {
    const int qi = i / 64, d = i % 64;
    qs[qi][d] = (q0 + qi < T && d < dh) ? base[(size_t)(q0 + qi) * ld + d] : 0.f;
  }
  float mx[kAttnQ / kAttnWarps], l[kAttnQ / kAttnWarps], o0[kAttnQ / kAttnWarps], o1[kAttnQ / kAttnWarps];
#pragma unroll
  for (int u = 0; u < kAttnQ / kAttnWarps; ++u) {
    mx[u] = -INFINITY;
    l[u] = 0.f;
    o0[u] = o1[u] = 0.f;
  }
  for (int j0 = 0; j0 < T; j0 += kAttnKeys) {
    __syncthreads();
    for (int i = threadIdx.x; i < kAttnKeys * 64; i += blockDim.x) {
      const int j = i / 64, d = i % 64;
      const bool in = j0 + j < T && d < dh;
      ks[j][d] = in ? base[(size_t)(j0 + j) * ld + H + d] : 0.f;
      vs[j][d] = in ? base[(size_t)(j0 + j) * ld + 2 * H + d] : 0.f;
    }
    __syncthreads();
    const int j = j0 + lane;
    const bool valid = j < T && (!any || mrow[j] != 0);
#pragma unroll
    for (int u = 0; u < kAttnQ / kAttnWarps; ++u) {
      const int qi = warp + kAttnWarps * u;
      float s = 0.f;
      for (int d = 0; d < dh; ++d) s = fmaf(qs[qi][d], ks[lane][d], s);
      s = valid ? (any ? s * scale : 0.f) : -INFINITY;
      float cm = s;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) cm = fmaxf(cm, __shfl_xor_sync(0xffffffffu, cm, o));
      const float mnew = fmaxf(mx[u], cm);
      if (mnew == -INFINITY) continue;  // nothing unmasked yet
      const float corr = expf(mx[u] - mnew);
      const float pj = valid ? expf(s - mnew) : 0.f;
      l[u] = l[u] * corr + warp_sum(pj);
      float a0 = o0[u] * corr, a1 = o1[u] * corr;
      for (int jj = 0; jj < kAttnKeys; ++jj) {
        const float pb = __shfl_sync(0xffffffffu, pj, jj);
        a0 = fmaf(pb, vs[jj][lane], a0);
        a1 = fmaf(pb, vs[jj][lane + 32], a1);
      }
      o0[u] = a0;
      o1[u] = a1;
      mx[u] = mnew;
    }
  }
  const int Hp = kpad(H);
#pragma unroll
  for (int u = 0; u < kAttnQ / kAttnWarps; ++u) {
    const int t = q0 + warp + kAttnWarps * u;
    if (t >= T) continue;
    __nv_bfloat16* row = ctx + ((size_t)b * T + t) * 2 * Hp + (size_t)h * dh;
    const float inv = 1.0f / l[u];
    if (lane < dh) store_split(row, Hp, lane, o0[u] * inv);
    if (lane + 32 < dh) store_split(row, Hp, lane + 32, o1[u] * inv);
  }
}

// W f32 [N, K] -> Ws bf16 [N, 2 Kp] hi | lo (zero K tail)
__global__ void split_weight_kernel(const float* __restrict__ W, int N, int K, __nv_bfloat16* __restrict__ Ws) {
  const int Kp = kpad(K);
  const int64_t total = (int64_t)N * Kp;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t n = i / Kp;
    const int k = (int)(i % Kp);
    store_split(Ws + n * 2 * Kp, Kp, k, k < K ? W[n * K + k] : 0.f);
  }
}

}  // namespace

// ------------------------------------------------------------------------------------------- model
namespace text {

struct DevLinear {
  int K = 0, N = 0;
  DevBuf<__nv_bfloat16> ws;  // [N, 2 Kp]
  DevBuf<float> b;
  alignas(64) unsigned char map[128];
};

struct DevLN {
  DevBuf<float> g, b;
  float eps = 0.f;
};

struct DevLayer {
  DevLinear qkv, o, f1, f2;
  DevLN ln1, ln2;
  float scale = 0.f;
};

// one GEMM of the plan: its tiles, K slices and the A operand's map
struct Gemm {
  const DevLinear* w = nullptr;
  int M = 0, tiles_n = 0, tiles_m = 0, splits = 1;
  alignas(64) unsigned char map_a[128];
};

// Everything fixed by (B, T): buffers, the K split of every GEMM and the operand maps
struct Plan {
  int B = 0, T = 0;
  DevBuf<int64_t> ids, mask;
  DevBuf<float> h0, h1, qkv, P, out;
  DevBuf<__nv_bfloat16> hs, ctx, fs, ps, p1s;
  Gemm g_qkv, g_o, g_f1, g_f2, g_pool, g_p1, g_p2;
};

}  // namespace text
}  // namespace am

struct am_text_model {
  am::text::Program prog;  // host copy released after upload, except the shapes
  int L = 0, H = 0, heads = 0, dh = 0, ffn = 0, vocab = 0, max_pos = 0, pad_id = 0, out_dim = 0;
  bool sdpa = false, mask_where = false;
  am::DevBuf<float> word, pos, type_row;
  am::text::DevLN emb_ln;
  std::vector<std::unique_ptr<am::text::DevLayer>> layers;
  am::text::DevLinear pool, p1, p2;
  std::unique_ptr<am::text::Plan> plan;
  am::Stream stream;
};

namespace am {
namespace {

using text::DevLinear;
using text::DevLN;
using text::Gemm;
using text::Plan;

int upload(DevBuf<float>& d, const std::vector<float>& h, cudaStream_t st) {
  AM_TRY(d.alloc(h.size()));
  if (!h.empty()) AM_CUDA(cudaMemcpyAsync(d.p, h.data(), h.size() * 4, cudaMemcpyHostToDevice, st));
  return AM_OK;
}

int upload_linear(DevLinear& d, const Linear& l, cudaStream_t st) {
  d.K = l.K;
  d.N = l.N;
  const int Kp = kpad(l.K);
  DevBuf<float> w;
  AM_TRY(upload(w, l.w, st));
  AM_TRY(d.ws.alloc((size_t)l.N * 2 * Kp));
  AM_LAUNCH(split_weight_kernel, grid_for((int64_t)l.N * Kp), 256, 0, st, w.p, l.N, l.K, d.ws.p);
  AM_CUDA(cudaStreamSynchronize(st));
  std::vector<float> b = l.b;
  if (b.empty()) b.assign((size_t)l.N, 0.f);
  AM_TRY(upload(d.b, b, st));
  return gemm::encode_map_bf16(d.map, d.ws.p, 2 * Kp, l.N, 2 * Kp, kTileN);
}

int upload_ln(DevLN& d, const LN& l, cudaStream_t st) {
  d.eps = l.eps;
  AM_TRY(upload(d.g, l.g, st));
  return upload(d.b, l.b, st);
}

// the K split of one GEMM.  linear_kernel holds one CTA per SM, so a wave is sm_count() CTAs.  When the tiles alone
// fill at least one wave, each tile runs whole K.  Otherwise K is cut into floor(SMs / tiles) balanced slices of
// whole 64-wide chunks (at most one per chunk): the most CTAs that still run as one wave.  A single query (M = 77) on
// 132 SMs: Q|K|V (N = 2304, 36 tiles) 3 slices of 4 chunks, 108 CTAs; output projection and pooler (N = 768, 12 tiles)
// 11 slices of 1-2 chunks, 132 CTAs; FFN up (N = 3072, 48 tiles) 2 slices of 6, 96 CTAs; FFN down (K = 3072, 12
// tiles) 11 slices of 4-5 chunks, 132 CTAs.  More slices would need a second wave and lengthen the slowest SM's
// chunk count: 144 one-chunk CTAs for the output projection take two waves, as long as 132 CTAs of up to 2 chunks.
int plan_gemm(Gemm& g, const DevLinear& w, int M, const void* a_base, int64_t a_rows, int64_t a_pitch) {
  g.w = &w;
  g.M = M;
  g.tiles_n = ceil_div(w.N, kTileN);
  g.tiles_m = ceil_div(M, kTileM);
  const int num_kb = kpad(w.K) / kChunkK;
  const int tiles = g.tiles_n * g.tiles_m;
  g.splits = tiles >= sm_count() ? 1 : std::max(1, std::min(num_kb, sm_count() / tiles));
  return gemm::encode_map_bf16(g.map_a, a_base, 2 * kpad(w.K), a_rows, a_pitch, kTileM);
}

size_t gemm_ws(const Gemm& g) { return (size_t)g.splits * g.M * g.w->N; }

int run_gemm(const Gemm& g, cudaStream_t st, float* P) {
  AM_TRY(allow_dynamic_smem<linear_kernel>(kLinearSmem));
  const dim3 grid(g.tiles_n, g.tiles_m, g.splits);
  AM_LAUNCH(linear_kernel, grid, pipe::kThreads, kLinearSmem, st, *reinterpret_cast<const CUtensorMap*>(g.map_a),
            *reinterpret_cast<const CUtensorMap*>(g.w->map), g.M, g.w->N, kpad(g.w->K), P);
  return AM_OK;
}

int run_epilogue(const Gemm& g, EpiArgs a, cudaStream_t st, const float* P) {
  a.P = P;
  a.splits = g.splits;
  a.M = g.M;
  a.N = g.w->N;
  a.bias = g.w->b.p;
  AM_LAUNCH(row_epilogue_kernel, g.M, kRowThreads, (size_t)a.N * sizeof(float), st, a);
  return AM_OK;
}

int make_plan(am_text_model* m, int B, int T) {
  auto pl = std::make_unique<Plan>();
  Plan& p = *pl;
  p.B = B;
  p.T = T;
  const int M = B * T, H = m->H, Hp = kpad(H), Fp = kpad(m->ffn), P1p = kpad(m->p1.N);
  AM_TRY(p.ids.alloc((size_t)M));
  AM_TRY(p.mask.alloc((size_t)M));
  AM_TRY(p.h0.alloc((size_t)M * H));
  AM_TRY(p.h1.alloc((size_t)M * H));
  AM_TRY(p.qkv.alloc((size_t)M * 3 * H));
  AM_TRY(p.hs.alloc((size_t)M * 2 * Hp));
  AM_TRY(p.ctx.alloc((size_t)M * 2 * Hp));
  // attention writes columns [0, H) of each half; the K tail [H, Hp) the output projection reads stays zero
  AM_CUDA(cudaMemsetAsync(p.ctx.p, 0, (size_t)M * 2 * Hp * sizeof(__nv_bfloat16), m->stream.s));
  AM_TRY(p.fs.alloc((size_t)M * 2 * Fp));
  AM_TRY(p.ps.alloc((size_t)B * 2 * Hp));
  AM_TRY(p.p1s.alloc((size_t)B * 2 * P1p));
  AM_TRY(p.out.alloc((size_t)B * m->out_dim));
  const text::DevLayer& L0 = *m->layers[0];
  AM_TRY(plan_gemm(p.g_qkv, L0.qkv, M, p.hs.p, M, 2 * Hp));
  AM_TRY(plan_gemm(p.g_o, L0.o, M, p.ctx.p, M, 2 * Hp));
  AM_TRY(plan_gemm(p.g_f1, L0.f1, M, p.hs.p, M, 2 * Hp));
  AM_TRY(plan_gemm(p.g_f2, L0.f2, M, p.fs.p, M, 2 * Fp));
  // the pooler reads token 0 of every batch row straight from the split hidden state: B rows T rows apart
  AM_TRY(plan_gemm(p.g_pool, m->pool, B, p.hs.p, B, (int64_t)T * 2 * Hp));
  AM_TRY(plan_gemm(p.g_p1, m->p1, B, p.ps.p, B, 2 * Hp));
  AM_TRY(plan_gemm(p.g_p2, m->p2, B, p.p1s.p, B, 2 * P1p));
  size_t ws = 0;
  for (const Gemm* g : {&p.g_qkv, &p.g_o, &p.g_f1, &p.g_f2, &p.g_pool, &p.g_p1, &p.g_p2}) ws = std::max(ws, gemm_ws(*g));
  AM_TRY(p.P.alloc(ws));
  m->plan = std::move(pl);
  return AM_OK;
}

// the same Gemm over another layer's weights (every layer has the same shapes, so the same split and A map)
Gemm with_weights(const Gemm& g, const DevLinear& w) {
  Gemm r = g;
  r.w = &w;
  return r;
}

int forward(am_text_model* m, cudaStream_t st) {
  Plan& p = *m->plan;
  const int M = p.B * p.T, H = m->H;
  AM_LAUNCH(embed_ln_kernel, M, kRowThreads, (size_t)H * sizeof(float), st, p.ids.p, p.T, H, m->pad_id, m->word.p,
            m->pos.p, m->type_row.p, m->emb_ln.g.p, m->emb_ln.b.p, m->emb_ln.eps, p.h0.p, p.hs.p);
  for (const auto& lp : m->layers) {
    const text::DevLayer& L = *lp;
    EpiArgs e;
    // Q | K | V
    const Gemm gq = with_weights(p.g_qkv, L.qkv);
    AM_TRY(run_gemm(gq, st, p.P.p));
    e.out = p.qkv.p;
    AM_TRY(run_epilogue(gq, e, st, p.P.p));
    const dim3 ag(ceil_div(p.T, kAttnQ), m->heads, p.B);
    AM_LAUNCH(attention_kernel, ag, kAttnWarps * 32, 0, st, p.qkv.p, p.mask.p, p.T, H, m->heads, m->dh, L.scale,
              p.ctx.p);
    // output projection + residual + LayerNorm
    const Gemm go = with_weights(p.g_o, L.o);
    AM_TRY(run_gemm(go, st, p.P.p));
    e = EpiArgs();
    e.residual = p.h0.p;
    e.ln_g = L.ln1.g.p;
    e.ln_b = L.ln1.b.p;
    e.eps = L.ln1.eps;
    e.out = p.h1.p;
    e.out_split = p.hs.p;
    AM_TRY(run_epilogue(go, e, st, p.P.p));
    // FFN
    const Gemm g1 = with_weights(p.g_f1, L.f1);
    AM_TRY(run_gemm(g1, st, p.P.p));
    e = EpiArgs();
    e.act = text::kGelu;
    e.out_split = p.fs.p;
    AM_TRY(run_epilogue(g1, e, st, p.P.p));
    const Gemm g2 = with_weights(p.g_f2, L.f2);
    AM_TRY(run_gemm(g2, st, p.P.p));
    e = EpiArgs();
    e.residual = p.h1.p;
    e.ln_g = L.ln2.g.p;
    e.ln_b = L.ln2.b.p;
    e.eps = L.ln2.eps;
    e.out = p.h0.p;
    e.out_split = p.hs.p;
    AM_TRY(run_epilogue(g2, e, st, p.P.p));
  }
  // pooler, projection, normalise
  EpiArgs e;
  AM_TRY(run_gemm(p.g_pool, st, p.P.p));
  e.act = text::kTanh;
  e.out_split = p.ps.p;
  AM_TRY(run_epilogue(p.g_pool, e, st, p.P.p));
  AM_TRY(run_gemm(p.g_p1, st, p.P.p));
  e = EpiArgs();
  e.act = text::kRelu;
  e.out_split = p.p1s.p;
  AM_TRY(run_epilogue(p.g_p1, e, st, p.P.p));
  AM_TRY(run_gemm(p.g_p2, st, p.P.p));
  e = EpiArgs();
  e.l2 = m->prog.normalize;
  e.out = p.out.p;
  AM_TRY(run_epilogue(p.g_p2, e, st, p.P.p));
  return AM_OK;
}

int lower_text(const void* data, size_t nbytes, const char* path, Program* prog) {
  OGraph g;
  AM_TRY(parse_model(data, nbytes, dir_of(path), &g));
  TextLowerer lw(g, *prog);
  return lw.run();
}

int read_whole(const char* path, std::vector<uint8_t>* buf, const char* who) {
  FILE* f = std::fopen(path, "rb");
  if (!f) {
    set_error("%s: cannot open %s", who, path);
    return AM_ERR_IO;
  }
  std::fseek(f, 0, SEEK_END);
  const long n = std::ftell(f);
  std::fseek(f, 0, SEEK_SET);
  buf->resize((size_t)std::max<long>(n, 0));
  const size_t got = n > 0 ? std::fread(buf->data(), 1, (size_t)n, f) : 0;
  std::fclose(f);
  if (n <= 0 || got != (size_t)n) {
    set_error("%s: short read on %s", who, path);
    return AM_ERR_IO;
  }
  return AM_OK;
}

std::string describe(const Program& p) {
  char line[512];
  std::string o;
  const text::Layer& L0 = p.layers[0];
  std::snprintf(line, sizeof line,
                "text model: %zu layers; hidden %d; heads %d x %d; ffn %d; vocab %d; positions %d; pad id %d; "
                "embedding ln eps %g\n",
                p.layers.size(), p.H, p.heads, p.dh, p.ffn, p.vocab, p.max_pos, p.pad_id, p.emb_ln.eps);
  o += line;
  std::snprintf(line, sizeof line, "attention: %s scaling, score scale %.9g, %s mask\n",
                L0.sdpa ? "sdpa (Q and K^T scaled)" : "eager (scores scaled)", L0.scale,
                L0.mask_where ? "masked_fill (Where)" : "arithmetic (Sub/Mul)");
  o += line;
  for (size_t i = 0; i < p.layers.size(); ++i) {
    const text::Layer& l = p.layers[i];
    std::snprintf(line, sizeof line, "L%-3zu qkv %d->%d  out %d->%d +res ln(eps %g)  ffn %d->%d gelu  %d->%d +res ln(eps %g)\n",
                  i, l.qkv.K, l.qkv.N, l.o.K, l.o.N, l.ln1.eps, l.f1.K, l.f1.N, l.f2.K, l.f2.N, l.ln2.eps);
    o += line;
  }
  std::snprintf(line, sizeof line, "pooler token 0 %d->%d tanh; projection %d->%d relu %d->%d; %s\n", p.pool.K, p.pool.N,
                p.p1.K, p.p1.N, p.p2.K, p.p2.N, p.normalize ? "l2 normalise" : "no normalise");
  o += line;
  return o;
}

int finish_text_load(Program&& prog, am_text_model** out) {
  AM_TRY(ensure_init());
  if (!gemm::available()) {
    set_error("am_text_load: the wgmma GEMM path is unavailable on this device; no fallback is shipped");
    return AM_ERR_NO_DEVICE;
  }
  std::unique_ptr<am_text_model> m(new am_text_model());
  AM_TRY(m->stream.create());
  const cudaStream_t st = m->stream.s;
  m->L = (int)prog.layers.size();
  m->H = prog.H;
  m->heads = prog.heads;
  m->dh = prog.dh;
  m->ffn = prog.ffn;
  m->vocab = prog.vocab;
  m->max_pos = prog.max_pos;
  m->pad_id = prog.pad_id;
  m->out_dim = prog.out_dim();
  m->sdpa = prog.layers[0].sdpa;
  m->mask_where = prog.layers[0].mask_where;
  AM_TRY(upload(m->word, prog.word, st));
  AM_TRY(upload(m->pos, prog.pos, st));
  AM_TRY(upload(m->type_row, prog.type_row, st));
  AM_TRY(upload_ln(m->emb_ln, prog.emb_ln, st));
  for (const text::Layer& l : prog.layers) {
    auto d = std::make_unique<text::DevLayer>();
    AM_TRY(upload_linear(d->qkv, l.qkv, st));
    AM_TRY(upload_linear(d->o, l.o, st));
    AM_TRY(upload_linear(d->f1, l.f1, st));
    AM_TRY(upload_linear(d->f2, l.f2, st));
    AM_TRY(upload_ln(d->ln1, l.ln1, st));
    AM_TRY(upload_ln(d->ln2, l.ln2, st));
    d->scale = l.scale;
    m->layers.push_back(std::move(d));
  }
  AM_TRY(upload_linear(m->pool, prog.pool, st));
  AM_TRY(upload_linear(m->p1, prog.p1, st));
  AM_TRY(upload_linear(m->p2, prog.p2, st));
  AM_CUDA(cudaStreamSynchronize(st));
  // keep the shapes and flags, drop the host weights
  m->prog.normalize = prog.normalize;
  *out = m.release();
  return AM_OK;
}

}  // namespace
}  // namespace am

using namespace am;

extern "C" int am_text_load_mem(const void* blob, size_t nbytes, am_text_model** out) {
  AM_CHECK(out != nullptr, "am_text_load_mem: out is NULL");
  *out = nullptr;
  AM_CHECK(blob != nullptr && nbytes >= 20, "am_text_load_mem: empty blob");
  text::Program prog;
  AM_TRY(lower_text(blob, nbytes, nullptr, &prog));
  return finish_text_load(std::move(prog), out);
}

extern "C" int am_text_load(const char* path, am_text_model** out) {
  AM_CHECK(out != nullptr && path != nullptr, "am_text_load: NULL argument");
  *out = nullptr;
  text::Program prog;
  {
    std::vector<uint8_t> buf;
    AM_TRY(read_whole(path, &buf, "am_text_load"));
    AM_TRY(lower_text(buf.data(), buf.size(), path, &prog));
  }
  return finish_text_load(std::move(prog), out);
}

extern "C" int am_text_describe_file(const char* path, char* buf, int cap) {
  AM_CHECK(path != nullptr, "am_text_describe_file: NULL path");
  std::vector<uint8_t> data;
  AM_TRY(read_whole(path, &data, "am_text_describe_file"));
  text::Program prog;
  AM_TRY(lower_text(data.data(), data.size(), path, &prog));
  const std::string d = describe(prog);
  if (buf && cap > 0) {
    const size_t n = std::min((size_t)cap - 1, d.size());
    std::memcpy(buf, d.data(), n);
    buf[n] = 0;
  }
  return (int)d.size() + 1;
}

extern "C" int am_text_embedding_dim(const am_text_model* m) { return m ? m->out_dim : 0; }

extern "C" int am_text_release_workspace(am_text_model* m) {
  AM_CHECK(m != nullptr, "am_text_release_workspace: NULL model");
  AM_CUDA(cudaStreamSynchronize(m->stream.s));
  m->plan.reset();
  return AM_OK;
}

extern "C" void am_text_free(am_text_model* m) {
  if (m) cudaStreamSynchronize(m->stream.s);
  delete m;
}

extern "C" int am_text_embed(am_text_model* m, const int64_t* ids, const int64_t* mask, int B, int T, float* out) {
  AM_CHECK(m != nullptr && ids != nullptr && mask != nullptr && out != nullptr, "am_text_embed: NULL argument");
  AM_CHECK(B >= 1 && T >= 1, "am_text_embed: B = %d, T = %d", B, T);
  // RoBERTa's largest position id is T + pad
  AM_CHECK(T + m->pad_id < m->max_pos, "am_text_embed: T = %d exceeds the model's %d positions (pad id %d)", T,
           m->max_pos, m->pad_id);
  for (int64_t i = 0; i < (int64_t)B * T; ++i)
    AM_CHECK(ids[i] >= 0 && ids[i] < m->vocab, "am_text_embed: token id %lld at %lld outside [0, %d)", (long long)ids[i],
             (long long)i, m->vocab);
  const cudaStream_t st = m->stream.s;
  if (!m->plan || m->plan->B != B || m->plan->T != T) {
    AM_CUDA(cudaStreamSynchronize(st));
    m->plan.reset();
    AM_TRY(make_plan(m, B, T));
  }
  text::Plan& p = *m->plan;
  const size_t n = (size_t)B * T;
  AM_CUDA(cudaMemcpyAsync(p.ids.p, ids, n * 8, cudaMemcpyHostToDevice, st));
  AM_CUDA(cudaMemcpyAsync(p.mask.p, mask, n * 8, cudaMemcpyHostToDevice, st));
  AM_TRY(forward(m, st));
  AM_CUDA(cudaMemcpyAsync(out, p.out.p, (size_t)B * m->out_dim * 4, cudaMemcpyDeviceToHost, st));
  AM_CUDA(cudaStreamSynchronize(st));
  return AM_OK;
}
