// AMW1 weight blob (audiomuse-ai_b200/weights.py) -> ModelSpec.
#include "common.cuh"
#include "model_spec.cuh"

namespace am {

namespace {

struct Reader {
  const uint8_t* p;
  const uint8_t* end;
  bool ok = true;
  template <typename T>
  T get() {
    T v{};
    if (p + sizeof(T) > end) {
      ok = false;
      return v;
    }
    std::memcpy(&v, p, sizeof(T));
    p += sizeof(T);
    return v;
  }
  std::vector<float> floats() {
    const uint64_t n = get<uint64_t>();
    std::vector<float> v;
    if (!ok || n > (uint64_t)(end - p) / 4) {
      ok = false;
      return v;
    }
    v.resize(n);
    std::memcpy(v.data(), p, n * 4);
    p += n * 4;
    return v;
  }
};

}  // namespace

int load_amw1_spec(const void* blob, size_t nbytes, ModelSpec* spec) {
  Reader r{(const uint8_t*)blob, (const uint8_t*)blob + nbytes};
  char magic[4];
  for (int i = 0; i < 4; ++i) magic[i] = (char)r.get<uint8_t>();
  if (!r.ok || std::memcmp(magic, "AMW1", 4) != 0) {
    set_error("weights: bad magic (expected AMW1 or an ONNX ModelProto)");
    return AM_ERR_IO;
  }
  const uint32_t version = r.get<uint32_t>();
  spec->n_mels = (int)r.get<uint32_t>();
  spec->emb = (int)r.get<uint32_t>();
  spec->source = "AMW1";
  const uint32_t n_layers = r.get<uint32_t>();
  if (!r.ok || version != 1 || n_layers == 0 || n_layers > 4096) {
    set_error("weights: bad header (version %u, %u layers)", version, n_layers);
    return AM_ERR_IO;
  }
  for (uint32_t li = 0; li < n_layers; ++li) {
    const uint32_t type = r.get<uint32_t>();
    int32_t prm[8];
    for (int i = 0; i < 8; ++i) prm[i] = r.get<int32_t>();
    if (!r.ok) break;
    if (type == kHead) {  // pn_block (1x1 stride s) -> mean -> Projection -> LayerNorm -> L2 as a row program
      const int cin = prm[0], trunk = prm[1], emb = prm[2], stride = prm[3];
      float ln_eps;
      std::memcpy(&ln_eps, &prm[4], 4);
      auto pn_w = r.floats(), pn_b = r.floats(), l1 = r.floats(), l2 = r.floats(), g = r.floats(), b = r.floats();
      if (!r.ok || pn_w.size() != (size_t)trunk * cin || pn_b.size() != (size_t)trunk || l1.size() != (size_t)emb * trunk ||
          l2.size() != (size_t)emb * emb || g.size() != (size_t)emb || b.size() != (size_t)emb) {
        set_error("weights: malformed head record");
        return AM_ERR_IO;
      }
      auto reg = [&](int dim) {
        spec->reg_dim.push_back(dim);
        return spec->n_regs++;
      };
      VecOp pool;
      pool.kind = kVecPool;
      pool.stride = stride;
      pool.N = cin;
      pool.dst = reg(cin);
      VecOp pn;
      pn.kind = kVecLinear;
      pn.a = pool.dst;
      pn.K = cin;
      pn.N = trunk;
      pn.w = pn_w;
      pn.bias = pn_b;
      pn.dst = reg(trunk);
      VecOp e1;
      e1.kind = kVecLinear;
      e1.a = pn.dst;
      e1.K = trunk;
      e1.N = emb;
      e1.w = l1;
      e1.dst = reg(emb);
      VecOp e2;
      e2.kind = kVecLinear;
      e2.a = e1.dst;
      e2.K = emb;
      e2.N = emb;
      e2.act = kActGelu;
      e2.w = l2;
      e2.dst = reg(emb);
      VecOp fin;
      fin.kind = kVecAddLnL2;
      fin.a = e1.dst;
      fin.b = e2.dst;
      fin.N = emb;
      fin.eps = ln_eps;
      fin.eps2 = 1e-12f;
      fin.w = g;
      fin.bias = b;
      fin.dst = reg(emb);
      spec->head = {pool, pn, e1, e2, fin};
      continue;
    }
    LayerSpec L;
    L.type = (int)type;
    if (type == kStem) {
      L.cin = 1;
      L.cout = prm[0];
      L.kh = L.kw = 3;
      L.stride = 2;
      L.act = kActRelu6;
      L.pad_t = prm[1];
      L.pad_b = prm[2];
      L.pad_l = prm[3];
      L.pad_r = prm[4];
      L.aux0 = r.floats();
      L.aux1 = r.floats();
      L.w = r.floats();
      L.aux2 = r.floats();
      L.bias = r.floats();
      if (!r.ok || L.aux0.size() != (size_t)spec->n_mels || L.aux1.size() != (size_t)spec->n_mels || L.w.size() != 9 ||
          L.aux2.size() != (size_t)L.cout || L.bias.size() != (size_t)L.cout) {
        set_error("weights: malformed stem record");
        return AM_ERR_IO;
      }
    } else if (type == kPointwise) {
      L.cin = prm[0];
      L.cout = prm[1];
      L.act = prm[2];
      L.residual = prm[3];
      L.block_start = prm[4];
      L.w = r.floats();
      L.bias = r.floats();
      if (!r.ok || L.w.size() != (size_t)L.cin * L.cout || L.bias.size() != (size_t)L.cout) {
        set_error("weights: malformed pointwise record (layer %u)", li);
        return AM_ERR_IO;
      }
    } else if (type == kDepthwise) {
      L.cin = L.cout = prm[0];
      L.stride = prm[1];
      L.block_start = prm[4];
      L.kh = L.kw = 3;
      L.pad_t = L.pad_b = L.pad_l = L.pad_r = 1;
      L.act = kActRelu6;
      L.w = r.floats();
      L.bias = r.floats();  // w: [c, 9]
      if (!r.ok || L.w.size() != (size_t)L.cin * 9 || L.bias.size() != (size_t)L.cin || (L.stride != 1 && L.stride != 2)) {
        set_error("weights: malformed depthwise record (layer %u)", li);
        return AM_ERR_IO;
      }
    } else {
      set_error("weights: unknown layer type %u", type);
      return AM_ERR_IO;
    }
    spec->layers.push_back(std::move(L));
  }
  if (!r.ok) {
    set_error("weights: truncated blob");
    return AM_ERR_IO;
  }
  return AM_OK;
}

}  // namespace am
