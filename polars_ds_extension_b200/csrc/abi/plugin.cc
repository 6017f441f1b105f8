// Plugin layer: the `_polars_plugin_*` symbols Polars dlopen()s (see include/polars_plugin_abi.h).
//   import : SeriesExport / Arrow C data  ->  pdsb_column[] (zero-copy views of the Arrow buffers)
//   kwargs : pickle protocol <= 5 of a flat dict (what serde-pickle reads into LRKwargs / MultiLRKwargs / SWWLRKwargs,
//            /root/reference/src/num_ext/linear_regression.rs:27-66)
//   compute: pdsb_host_*  (lr_host.cc)
//   export : Arrow C data with the reference's names and nesting (LargeList "coeffs", Struct{pred,resid}, ...),
//            zero-copy over the pinned result buffers (released through the Arrow release callbacks).
#include "../common.h"
#include "../host/host.h"
#include "../../../include/polars_plugin_abi.h"
#include "../../../include/polars_plugin_num_abi.h"
#include "../../../include/polars_plugin_group_abi.h"
#include "../../../include/polars_plugin_group_logistic_abi.h"
#include <cstring>
#include <cstdlib>
#include <memory>
#include <map>
#include <vector>
#include <string>
#include <atomic>
#include <exception>
#include <thread>
#include <algorithm>

using namespace pdsb;

namespace {

// ------------------------------------------------------------------ pickle (flat dict) ----------------
struct PVal {
  enum Kind { NONE, BOOL, INT, FLOAT, STR, DICT, MARK } kind = NONE;
  bool b = false; int64_t i = 0; double f = 0.0; std::string s;
  std::shared_ptr<std::map<std::string, PVal>> d;
};

bool parse_pickle(const uint8_t* p, size_t n, std::map<std::string, PVal>& out) {
  std::vector<PVal> stack, memo;
  size_t pos = 0;
  auto need = [&](size_t k) { return k <= n - pos; };          // pos <= n always; no overflow for hostile lengths
  constexpr size_t MAX_MEMO = 1 << 16;                           // a flat kwargs dict memoises a few dozen objects
  auto rd_le = [&](size_t k) { uint64_t v = 0; for (size_t j = 0; j < k; ++j) v |= (uint64_t)p[pos + j] << (8 * j); pos += k; return v; };
  while (pos < n) {
    uint8_t op = p[pos++];
    switch (op) {
      case 0x80: if (!need(1)) return false; pos += 1; break;                  // PROTO
      case 0x95: if (!need(8)) return false; pos += 8; break;                  // FRAME
      case '}': { PVal v; v.kind = PVal::DICT; v.d = std::make_shared<std::map<std::string, PVal>>(); stack.push_back(v); break; }
      case 0x94: if (stack.empty() || memo.size() >= MAX_MEMO) return false; memo.push_back(stack.back()); break;   // MEMOIZE
      case 'q': if (!need(1) || stack.empty()) return false; { size_t k = p[pos++]; if (memo.size() <= k) memo.resize(k + 1); memo[k] = stack.back(); } break;
      case 'r': if (!need(4) || stack.empty()) return false; { size_t k = rd_le(4); if (k >= MAX_MEMO) return false; if (memo.size() <= k) memo.resize(k + 1); memo[k] = stack.back(); } break;
      case '(': { PVal v; v.kind = PVal::MARK; stack.push_back(v); break; }
      case 0x8c: { if (!need(1)) return false; size_t k = p[pos++]; if (!need(k)) return false; PVal v; v.kind = PVal::STR; v.s.assign((const char*)p + pos, k); pos += k; stack.push_back(v); break; }
      case 'X': { if (!need(4)) return false; size_t k = rd_le(4); if (!need(k)) return false; PVal v; v.kind = PVal::STR; v.s.assign((const char*)p + pos, k); pos += k; stack.push_back(v); break; }
      case 0x8d: { if (!need(8)) return false; size_t k = rd_le(8); if (!need(k)) return false; PVal v; v.kind = PVal::STR; v.s.assign((const char*)p + pos, k); pos += k; stack.push_back(v); break; }
      case 'J': { if (!need(4)) return false; PVal v; v.kind = PVal::INT; v.i = (int32_t)rd_le(4); stack.push_back(v); break; }
      case 'K': { if (!need(1)) return false; PVal v; v.kind = PVal::INT; v.i = p[pos++]; stack.push_back(v); break; }
      case 'M': { if (!need(2)) return false; PVal v; v.kind = PVal::INT; v.i = (int64_t)rd_le(2); stack.push_back(v); break; }
      case 0x8a: { if (!need(1)) return false; size_t k = p[pos++]; if (!need(k) || k > 8) return false;
                   uint64_t u = 0; for (size_t j = 0; j < k; ++j) u |= (uint64_t)p[pos + j] << (8 * j);
                   if (k > 0 && k < 8 && (p[pos + k - 1] & 0x80)) u |= ~uint64_t(0) << (8 * k);
                   pos += k; PVal v; v.kind = PVal::INT; v.i = (int64_t)u; stack.push_back(v); break; }
      case 'G': { if (!need(8)) return false; uint64_t u = 0; for (int j = 0; j < 8; ++j) u = (u << 8) | p[pos + j]; pos += 8;
                  PVal v; v.kind = PVal::FLOAT; memcpy(&v.f, &u, 8); stack.push_back(v); break; }
      case 0x88: { PVal v; v.kind = PVal::BOOL; v.b = true; stack.push_back(v); break; }
      case 0x89: { PVal v; v.kind = PVal::BOOL; v.b = false; stack.push_back(v); break; }
      case 'N': { PVal v; stack.push_back(v); break; }
      case 'h': { if (!need(1)) return false; size_t k = p[pos++]; if (k >= memo.size()) return false; stack.push_back(memo[k]); break; }
      case 'j': { if (!need(4)) return false; size_t k = rd_le(4); if (k >= memo.size()) return false; stack.push_back(memo[k]); break; }
      case 's': { if (stack.size() < 3) return false; PVal val = stack.back(); stack.pop_back(); PVal key = stack.back(); stack.pop_back();
                  if (stack.back().kind != PVal::DICT || key.kind != PVal::STR) return false; (*stack.back().d)[key.s] = val; break; }
      case 'u': { size_t m = stack.size(); while (m > 0 && stack[m - 1].kind != PVal::MARK) --m; if (m == 0 || m < 2) return false;
                  PVal& dict = stack[m - 2]; if (dict.kind != PVal::DICT) return false;
                  for (size_t j = m; j + 1 < stack.size(); j += 2) { if (stack[j].kind != PVal::STR) return false; (*dict.d)[stack[j].s] = stack[j + 1]; }
                  stack.resize(m - 1); break; }
      case '.': if (stack.empty() || stack.back().kind != PVal::DICT) return false; out = *stack.back().d; return true;
      default: return false;
    }
  }
  return false;
}

struct Kwargs {
  std::map<std::string, PVal> m;
  std::string null_policy, solver, std_err;
  pdsb_lr_kwargs k{};
  bool has(const char* key) const { return m.count(key) > 0; }
  double num(const char* key, double def) const {
    auto it = m.find(key); if (it == m.end()) return def;
    switch (it->second.kind) { case PVal::FLOAT: return it->second.f; case PVal::INT: return (double)it->second.i; case PVal::BOOL: return it->second.b; default: return def; }
  }
  int64_t integer(const char* key, int64_t def) const {
    auto it = m.find(key); if (it == m.end()) return def;
    switch (it->second.kind) { case PVal::INT: return it->second.i; case PVal::FLOAT: return (int64_t)it->second.f; case PVal::BOOL: return it->second.b; default: return def; }
  }
  std::string str(const char* key, const char* def) const {
    auto it = m.find(key); if (it == m.end() || it->second.kind != PVal::STR) return def; return it->second.s;
  }
};

// required keys mirror the non-#[serde(default)] fields of the reference structs
bool load_kwargs(const uint8_t* p, size_t n, Kwargs& kw, const char* const* required) {
  if (!p || n == 0 || !parse_pickle(p, n, kw.m)) { set_error("failed to decode the pickled kwargs"); return false; }
  for (const char* const* r = required; *r; ++r)
    if (!kw.has(*r)) { set_error("kwargs: missing field `%s`", *r); return false; }
  kw.null_policy = kw.str("null_policy", "raise");
  kw.solver = kw.str("solver", "qr");
  kw.std_err = kw.str("std_err", "");
  kw.k.bias = kw.integer("bias", 0) != 0;
  kw.k.null_policy = kw.null_policy.c_str();
  kw.k.solver = kw.solver.c_str();
  kw.k.std_err = kw.std_err.c_str();
  kw.k.l1_reg = kw.num("l1_reg", 0.0);
  kw.k.l2_reg = kw.num("l2_reg", 0.0);
  kw.k.tol = kw.num("tol", 0.0);
  kw.k.weighted = kw.integer("weighted", 0) != 0;
  kw.k.positive = kw.integer("positive", 0) != 0;
  kw.k.max_iter = kw.integer("max_iter", 0);
  kw.k.singular_x_tol = kw.num("singular_x_tol", 0.0);
  kw.k.last_target_idx = kw.integer("last_target_idx", 1);
  kw.k.n = kw.integer("n", 0);
  kw.k.lambda = kw.num("lambda", 0.0);
  kw.k.min_size = kw.integer("min_size", 0);
  return true;
}

const char* const REQ_LR[] = {"bias", "null_policy", "solver", "l1_reg", "l2_reg", "tol", nullptr};
const char* const REQ_MULTI[] = {"bias", "null_policy", "solver", "last_target_idx", "l2_reg", nullptr};
const char* const REQ_SWW[] = {"null_policy", "n", "bias", "lambda", "min_size", nullptr};
const char* const REQ_SPLINE[] = {"lambda", nullptr};     // SplineKwargs (splines.rs:11-14)
const char* const REQ_ISO[] = {"has_weights", "increasing", nullptr};   // IsotonicRegKwargs (isotonic_regression.rs)

// ------------------------------------------------------------------ import ---------------------------
// Ownership follows polars-ffi version_0 (import_series / export_series, crate polars-ffi 0.55.2):
//   * the callee owns every input SeriesExport.  import_series MOVES each chunk out of its box with ptr::read, keeps it
//     for as long as the Series lives and releases it through the ArrowArray's own callback; SeriesExport::release only
//     frees the boxes and the schema and never touches the arrays.  So here: every ArrowArray is moved into `moved`
//     (source marked released, Arrow-spec move), released by us when the call is over, and then the export is released.
struct Imported {
  std::vector<pdsb_column> cols;
  std::vector<std::vector<pdsb_chunk>> chunks;
  std::vector<std::string> names;
  std::vector<ArrowArray> moved;
  SeriesExport* raw = nullptr; size_t n = 0;
  ~Imported() {
    for (ArrowArray& a : moved) if (a.release) a.release(&a);
    for (size_t i = 0; i < n; ++i) if (raw[i].release) raw[i].release(&raw[i]);
  }
};

int dtype_from_format(const char* f) {
  if (!f || !f[0] || f[1]) return -1;
  switch (f[0]) {
    case 'f': return PDSB_F32; case 'g': return PDSB_F64; case 'c': return PDSB_I8; case 'C': return PDSB_U8;
    case 's': return PDSB_I16; case 'S': return PDSB_U16; case 'i': return PDSB_I32; case 'I': return PDSB_U32;
    case 'l': return PDSB_I64; case 'L': return PDSB_U64; case 'b': return PDSB_BOOL;
  }
  return -1;
}

bool import_inputs(SeriesExport* in, size_t n, Imported& im) {
  im.raw = in; im.n = n;
  im.cols.resize(n); im.chunks.resize(n); im.names.resize(n);
  size_t total_chunks = 0;
  for (size_t i = 0; i < n; ++i) total_chunks += in[i].arrays ? in[i].len : 0;
  im.moved.reserve(total_chunks);                       // pointers into `moved` stay valid
  for (size_t i = 0; i < n; ++i)
    for (size_t c = 0; in[i].arrays && c < in[i].len; ++c) {
      ArrowArray* src = in[i].arrays[c];
      if (!src) continue;
      im.moved.push_back(*src);
      src->release = nullptr;
    }
  size_t mv = 0;
  for (size_t i = 0; i < n; ++i) {
    SeriesExport& se = in[i];
    if (!se.field) { set_error("plugin input %zu has no schema", i); return false; }
    int dt = dtype_from_format(se.field->format);
    if (dt < 0) { set_error("All columns need to be numeric."); return false; }
    im.names[i] = se.field->name ? se.field->name : "";
    int64_t nulls = 0;
    for (size_t c = 0; c < se.len; ++c) {
      if (!se.arrays || !se.arrays[c]) { set_error("plugin input %zu has a null chunk", i); return false; }
      ArrowArray* a = &im.moved[mv++];
      pdsb_chunk ch;
      ch.validity = (a->n_buffers > 0 && a->null_count != 0) ? (const uint8_t*)a->buffers[0] : nullptr;
      ch.data = a->n_buffers > 1 ? a->buffers[1] : nullptr;
      ch.offset = a->offset; ch.length = a->length;
      if (a->null_count < 0) nulls = -1; else if (nulls >= 0) nulls += a->null_count;
      im.chunks[i].push_back(ch);
    }
    pdsb_column& col = im.cols[i];
    col.name = im.names[i].c_str(); col.dtype = dt; col.n_chunks = (int)im.chunks[i].size();
    col.chunks = im.chunks[i].data(); col.null_count = nulls;
  }
  return true;
}

// ------------------------------------------------------------------ export ---------------------------
std::atomic<int64_t> g_live_results{0};   // exported results whose buffers have not been released yet (tests)
struct SharedResult {
  pdsb_host_result r; std::atomic<int> refs{1};
  SharedResult() { memset(&r, 0, sizeof(r)); g_live_results.fetch_add(1); }
  ~SharedResult() { g_live_results.fetch_sub(1); }
};
void sr_unref(SharedResult* s) { if (s && s->refs.fetch_sub(1) == 1) { pdsb_host_result_free(&s->r); delete s; } }

struct Node {
  std::string format, name;
  int64_t length = 0, null_count = 0;
  std::vector<const void*> buffers;       // borrowed (from SharedResult) or owned (in `owned`)
  std::vector<void*> owned;               // malloc'd, freed on release
  std::vector<std::unique_ptr<Node>> children;
};

struct ArrPriv { std::vector<void*> owned; SharedResult* sr; const void** bufs; ArrowArray** kids; };
struct SchPriv { char* format; char* name; ArrowSchema** kids; };

void release_schema(ArrowSchema* s) {
  if (!s || !s->release) return;
  SchPriv* p = (SchPriv*)s->private_data;
  for (int64_t i = 0; i < s->n_children; ++i) { if (s->children[i]->release) s->children[i]->release(s->children[i]); free(s->children[i]); }
  free(p->kids); free(p->format); free(p->name); delete p;
  s->release = nullptr;
}
void release_array(ArrowArray* a) {
  if (!a || !a->release) return;
  ArrPriv* p = (ArrPriv*)a->private_data;
  for (int64_t i = 0; i < a->n_children; ++i) { if (a->children[i]->release) a->children[i]->release(a->children[i]); free(a->children[i]); }
  for (void* o : p->owned) free(o);
  free(p->bufs); free(p->kids); sr_unref(p->sr); delete p;
  a->release = nullptr;
}

void fill_schema(const Node& nd, ArrowSchema* s) {
  SchPriv* p = new SchPriv();
  p->format = strdup(nd.format.c_str()); p->name = strdup(nd.name.c_str());
  p->kids = nd.children.empty() ? nullptr : (ArrowSchema**)malloc(sizeof(ArrowSchema*) * nd.children.size());
  for (size_t i = 0; i < nd.children.size(); ++i) { p->kids[i] = (ArrowSchema*)calloc(1, sizeof(ArrowSchema)); fill_schema(*nd.children[i], p->kids[i]); }
  s->format = p->format; s->name = p->name; s->metadata = nullptr; s->flags = 2 /* nullable */;
  s->n_children = (int64_t)nd.children.size(); s->children = p->kids; s->dictionary = nullptr;
  s->release = release_schema; s->private_data = p;
}
void fill_array(Node& nd, ArrowArray* a, SharedResult* sr) {
  ArrPriv* p = new ArrPriv();
  p->owned = std::move(nd.owned); p->sr = sr; if (sr) sr->refs.fetch_add(1);
  p->bufs = (const void**)malloc(sizeof(void*) * (nd.buffers.size() ? nd.buffers.size() : 1));
  for (size_t i = 0; i < nd.buffers.size(); ++i) p->bufs[i] = nd.buffers[i];
  p->kids = nd.children.empty() ? nullptr : (ArrowArray**)malloc(sizeof(ArrowArray*) * nd.children.size());
  for (size_t i = 0; i < nd.children.size(); ++i) { p->kids[i] = (ArrowArray*)calloc(1, sizeof(ArrowArray)); fill_array(*nd.children[i], p->kids[i], sr); }
  a->length = nd.length; a->null_count = nd.null_count; a->offset = 0;
  a->n_buffers = (int64_t)nd.buffers.size(); a->n_children = (int64_t)nd.children.size();
  a->buffers = p->bufs; a->children = p->kids; a->dictionary = nullptr;
  a->release = release_array; a->private_data = p;
}

// Output: the importer (polars-ffi import_series) takes the ArrowArray by ptr::read — a bitwise copy that leaves
// `release` set in our box — and owns it from then on; it drops the SeriesExport right after, whose release callback
// (c_release_series_export in polars-ffi) frees the boxes and the schema only.  Calling the array's release here would
// free the buffers under the imported Series and be followed by a second release when that Series is dropped.
struct SePriv { ArrowSchema* field; ArrowArray** arrays; };
void release_series(SeriesExport* se) {
  if (!se || !se->private_data) return;
  SePriv* p = (SePriv*)se->private_data;
  if (p->field) { if (p->field->release) p->field->release(p->field); free(p->field); }
  if (p->arrays) { free(p->arrays[0]); free(p->arrays); }
  delete p;
  se->private_data = nullptr; se->release = nullptr; se->field = nullptr; se->arrays = nullptr; se->len = 0;
}

void export_series(Node& root, SharedResult* sr, SeriesExport* ret) {
  SePriv* p = new SePriv();
  p->field = (ArrowSchema*)calloc(1, sizeof(ArrowSchema));
  fill_schema(root, p->field);
  p->arrays = (ArrowArray**)malloc(sizeof(ArrowArray*));
  p->arrays[0] = (ArrowArray*)calloc(1, sizeof(ArrowArray));
  fill_array(root, p->arrays[0], sr);
  ret->field = p->field; ret->arrays = p->arrays; ret->len = 1; ret->release = release_series; ret->private_data = p;
}

// ---- node builders ----
// one byte per row (0/1) -> Arrow validity bitmap.  8 rows per step (multiply-gather of the low bits), row ranges
// spread over a few threads for long outputs (rolling / recursive: one validity entry per input row).
void bitmap_range(const uint8_t* valid, int64_t b0, int64_t b1 /* byte range of the bitmap */, int64_t n, uint8_t* bm, int64_t* ones) {
  int64_t cnt = 0;
  for (int64_t b = b0; b < b1; ++b) {
    const int64_t i = b << 3;
    uint8_t v = 0;
    if (i + 8 <= n) {
      uint64_t x; memcpy(&x, valid + i, 8);
      x = (x | (x >> 1) | (x >> 2) | (x >> 3) | (x >> 4) | (x >> 5) | (x >> 6) | (x >> 7)) & 0x0101010101010101ull;   // any non-zero byte -> 1
      v = (uint8_t)((x * 0x0102040810204080ull) >> 56);
    } else {
      for (int64_t k = i; k < n; ++k) if (valid[k]) v |= (uint8_t)(1u << (k & 7));
    }
    bm[b] = v;
    cnt += __builtin_popcount(v);
  }
  *ones = cnt;
}
uint8_t* bitmap_from_bytes(const uint8_t* valid, int64_t n, int64_t* null_count) {
  const int64_t nb = (n + 7) / 8;
  uint8_t* bm = (uint8_t*)calloc((size_t)(nb + 8), 1);
  const int nt = n >= (int64_t(1) << 22) ? (int)std::min<int64_t>(8, std::max(1u, std::thread::hardware_concurrency())) : 1;
  std::vector<int64_t> ones(nt, 0);
  if (nt == 1) bitmap_range(valid, 0, nb, n, bm, &ones[0]);
  else {
    std::vector<std::thread> th;
    for (int t = 0; t < nt; ++t) th.emplace_back(bitmap_range, valid, nb * t / nt, nb * (t + 1) / nt, n, bm, &ones[t]);
    for (auto& t : th) t.join();
  }
  int64_t tot = 0; for (int64_t o : ones) tot += o;
  *null_count = n - tot;
  return bm;
}
uint8_t* bitmap_const(int64_t n, bool v) {
  uint8_t* bm = (uint8_t*)malloc((size_t)((n + 7) / 8 + 8));
  memset(bm, v ? 0xff : 0x00, (size_t)((n + 7) / 8 + 8));
  return bm;
}

// primitive array over a borrowed buffer; valid (bytes) optional; all_null overrides
std::unique_ptr<Node> prim_node(const char* name, bool f32, const void* data, int64_t n, const uint8_t* valid, bool all_null) {
  auto nd = std::make_unique<Node>();
  nd->format = f32 ? "f" : "g"; nd->name = name; nd->length = n;
  const void* vbuf = nullptr;
  if (all_null) { uint8_t* bm = bitmap_const(n, false); nd->owned.push_back(bm); vbuf = bm; nd->null_count = n; }
  else if (valid) { int64_t nc; uint8_t* bm = bitmap_from_bytes(valid, n, &nc); nd->owned.push_back(bm); vbuf = bm; nd->null_count = nc; }
  nd->buffers = {vbuf, data};
  return nd;
}
// owned copy of a small f64/f32 vector
std::unique_ptr<Node> prim_node_copy(const char* name, bool f32, const double* vals, int64_t n) {
  auto nd = std::make_unique<Node>();
  nd->format = f32 ? "f" : "g"; nd->name = name; nd->length = n;
  void* buf = malloc((size_t)(n ? n : 1) * (f32 ? 4 : 8));
  for (int64_t i = 0; i < n; ++i) { if (f32) ((float*)buf)[i] = (float)vals[i]; else ((double*)buf)[i] = vals[i]; }
  nd->owned.push_back(buf);
  nd->buffers = {nullptr, buf};
  return nd;
}
// LargeList<T> with `rows` lists of `width` values each over a borrowed values buffer
std::unique_ptr<Node> list_node(const char* name, bool f32, const void* values, int64_t rows, int64_t width,
                                const uint8_t* valid, bool all_null) {
  auto nd = std::make_unique<Node>();
  nd->format = "+L"; nd->name = name; nd->length = rows;
  int64_t* offs = (int64_t*)malloc(sizeof(int64_t) * (size_t)(rows + 1));
  const void* vbuf = nullptr;
  if (all_null) {
    for (int64_t i = 0; i <= rows; ++i) offs[i] = 0;
    uint8_t* bm = bitmap_const(rows, false); nd->owned.push_back(bm); vbuf = bm; nd->null_count = rows;
    nd->children.push_back(prim_node("item", f32, nullptr, 0, nullptr, false));
    // zero-length child still needs a non-null data pointer for some consumers
    void* dummy = calloc(1, 8); nd->children[0]->owned.push_back(dummy); nd->children[0]->buffers[1] = dummy;
  } else {
    // keep the fixed stride: null rows own `width` (ignored) values, so the values buffer is exported as is
    for (int64_t i = 0; i <= rows; ++i) offs[i] = i * width;
    if (valid) { int64_t nc; uint8_t* bm = bitmap_from_bytes(valid, rows, &nc); nd->owned.push_back(bm); vbuf = bm; nd->null_count = nc; }
    nd->children.push_back(prim_node("item", f32, values, rows * width, nullptr, false));
  }
  nd->owned.push_back(offs);
  nd->buffers = {vbuf, offs};
  return nd;
}
std::unique_ptr<Node> struct_node(const char* name, int64_t length) {
  auto nd = std::make_unique<Node>();
  nd->format = "+s"; nd->name = name; nd->length = length; nd->buffers = {nullptr};
  return nd;
}
std::unique_ptr<Node> utf8_node(const char* name, const std::vector<std::string>& vals) {
  auto nd = std::make_unique<Node>();
  nd->format = "U"; nd->name = name; nd->length = (int64_t)vals.size();
  int64_t* offs = (int64_t*)malloc(sizeof(int64_t) * (vals.size() + 1));
  size_t total = 0; for (auto& s : vals) total += s.size();
  char* data = (char*)malloc(total ? total : 1);
  size_t pos = 0;
  for (size_t i = 0; i < vals.size(); ++i) { offs[i] = (int64_t)pos; memcpy(data + pos, vals[i].data(), vals[i].size()); pos += vals[i].size(); }
  offs[vals.size()] = (int64_t)pos;
  nd->owned.push_back(offs); nd->owned.push_back(data);
  nd->buffers = {nullptr, offs, data};
  return nd;
}

void fail(SeriesExport* ret) { if (ret) { ret->private_data = nullptr; ret->release = nullptr; } }

// schema-only field export
void field_out(ArrowSchema* out, Node& nd) { fill_schema(nd, out); }
std::unique_ptr<Node> schema_prim(const char* name, bool f32) { auto n = std::make_unique<Node>(); n->format = f32 ? "f" : "g"; n->name = name; return n; }
std::unique_ptr<Node> schema_list(const char* name, bool f32) { auto n = std::make_unique<Node>(); n->format = "+L"; n->name = name; n->children.push_back(schema_prim("item", f32)); return n; }

// ------------------------------------------------------------------ expression bodies -----------------
// Every expression: import the inputs, decode the kwargs (required == nullptr: the symbol takes none and Polars passes an
// empty buffer), run the host call into a shared result and export the node tree `build` makes of it.  With `borrow` the tree points into the result's pinned buffers: each exported array holds
// a reference and the last release frees them.  Without it the tree owns copies and the result is freed here.
template <typename Compute, typename Build>
void run_expr(SeriesExport* in, size_t n, const uint8_t* kwp, size_t kwn, SeriesExport* ret, const char* const* required,
              Compute compute, Build build, bool borrow = true) {
  fail(ret);
  Imported im;
  if (!import_inputs(in, n, im)) return;
  Kwargs kw;
  if (required && !load_kwargs(kwp, kwn, kw, required)) return;
  SharedResult* sr = new SharedResult();
  if (compute(im, kw, &sr->r)) { sr_unref(sr); return; }
  auto root = build(im, kw, sr->r);
  export_series(*root, borrow ? sr : nullptr, ret);
  sr_unref(sr);
}

void run_lr(SeriesExport* in, size_t n, const uint8_t* kwp, size_t kwn, SeriesExport* ret, bool f32, bool pred, bool rcond) {
  run_expr(in, n, kwp, kwn, ret, REQ_LR,
    [&](const Imported& im, const Kwargs& kw, pdsb_host_result* r) {
      return pdsb_host_lin_reg(im.cols.data(), (int)n, &kw.k, f32, 1, pred, rcond, r);
    },
    [&](const Imported&, const Kwargs&, const pdsb_host_result& r) {
      if (rcond) {
        auto root = struct_node("", 1);
        root->children.push_back(list_node("coeffs", f32, r.coeffs, 1, r.n_coef, nullptr, false));
        root->children.push_back(list_node("singular_values", f32, r.singular_values, 1, r.n_coef, nullptr, false));
        return root;
      }
      if (!pred) return list_node("coeffs", f32, r.coeffs, 1, r.n_coef, nullptr, r.gated);
      auto root = struct_node("", r.n_rows);
      root->children.push_back(prim_node("pred", f32, r.pred, r.n_rows, r.valid, r.gated));
      root->children.push_back(prim_node("resid", f32, r.resid, r.n_rows, r.valid, r.gated));
      return root;
    });
}

void run_multi(SeriesExport* in, size_t n, const uint8_t* kwp, size_t kwn, SeriesExport* ret, bool f32, bool pred) {
  run_expr(in, n, kwp, kwn, ret, REQ_MULTI,
    [&](const Imported& im, const Kwargs& kw, pdsb_host_result* r) {
      const int t = (int)kw.k.last_target_idx;
      if (t < 1 || (size_t)t >= n) { set_error("last_target_idx out of range"); return 1; }
      return pdsb_host_lin_reg(im.cols.data(), (int)n, &kw.k, f32, t, pred, 0, r);
    },
    [&](const Imported& im, const Kwargs& kw, const pdsb_host_result& r) {
      const int t = (int)kw.k.last_target_idx;
      const size_t esz = f32 ? 4 : 8;
      if (!pred) {
        auto root = struct_node("coeffs", 1);
        for (int k = 0; k < t; ++k)
          root->children.push_back(list_node(im.names[k].c_str(), f32, (const char*)r.coeffs + (size_t)k * r.n_coef * esz, 1, r.n_coef, nullptr, r.gated));
        return root;
      }
      auto root = struct_node("all_preds", r.n_rows);
      for (int k = 0; k < t; ++k) {
        std::string pn = im.names[k] + "_pred", rn = im.names[k] + "_resid";
        root->children.push_back(prim_node(pn.c_str(), f32, (const char*)r.pred + (size_t)k * r.n_rows * esz, r.n_rows, nullptr, r.gated));
        root->children.push_back(prim_node(rn.c_str(), f32, (const char*)r.resid + (size_t)k * r.n_rows * esz, r.n_rows, nullptr, r.gated));
      }
      return root;
    });
}

// the report is small: exported as owned copies, so the pinned result is freed before the call returns
void run_report(SeriesExport* in, size_t n, const uint8_t* kwp, size_t kwn, SeriesExport* ret, bool f32, bool weighted) {
  run_expr(in, n, kwp, kwn, ret, REQ_LR,
    [&](const Imported& im, const Kwargs& kw, pdsb_host_result* r) {
      return pdsb_host_report(im.cols.data(), (int)n, &kw.k, f32, weighted, r);
    },
    [&](const Imported& im, const Kwargs& kw, const pdsb_host_result& r) {
      const int q = r.n_coef;
      std::vector<std::string> names;
      for (size_t i = weighted ? 3 : 2; i < n; ++i) names.push_back(im.names[i]);
      if (kw.k.bias) names.push_back("__bias__");
      static const char* se_names[] = {"std_err", "hc0_se", "hc1_se", "hc2_se", "hc3_se"};
      const char* se_name = weighted ? "std_err" : se_names[se_type_from_string(kw.k.std_err)];
      auto root = struct_node("lin_reg_report", q);
      root->children.push_back(utf8_node("features", names));
      const char* cn[8] = {"beta", se_name, "t", "p>|t|", "0.025", "0.975", "r2", "adj_r2"};
      for (int c = 0; c < 8; ++c) root->children.push_back(prim_node_copy(cn[c], f32, r.report + (size_t)c * q, q));
      return root;
    },
    false);
}

void run_online(SeriesExport* in, size_t n, const uint8_t* kwp, size_t kwn, SeriesExport* ret, bool f32, bool rolling) {
  run_expr(in, n, kwp, kwn, ret, REQ_SWW,
    [&](const Imported& im, const Kwargs& kw, pdsb_host_result* r) {
      return pdsb_host_online(im.cols.data(), (int)n, &kw.k, f32, rolling, r);
    },
    [&](const Imported&, const Kwargs&, const pdsb_host_result& r) {
      auto root = struct_node("", r.n_rows);
      root->children.push_back(list_node("coeffs", f32, r.coeffs, r.n_rows, r.n_coef, r.valid, false));
      root->children.push_back(prim_node("pred", f32, r.pred, r.n_rows, r.valid, false));
      return root;
    });
}

// pl_logistic_coeffs / pl_logistic_pred (logistic_regression.rs:10-99): LRKwargs, Float64 outputs
void run_logistic(SeriesExport* in, size_t n, const uint8_t* kwp, size_t kwn, SeriesExport* ret, bool pred) {
  run_expr(in, n, kwp, kwn, ret, REQ_LR,
    [&](const Imported& im, const Kwargs& kw, pdsb_host_result* r) {
      return pdsb_host_logistic(im.cols.data(), (int)n, &kw.k, pred, r);
    },
    [&](const Imported&, const Kwargs&, const pdsb_host_result& r) {
      if (!pred) return list_node("coeffs", false, r.coeffs, 1, r.n_coef, nullptr, false);
      return prim_node("pred", false, r.pred, r.n_rows, r.valid, false);
    });
}

// input 0 of the grouped symbols: the group offsets, one non-null Int64 chunk; then a target and the features
int group_offsets(const Imported& im, size_t n, const char* sym, const int64_t** offs, int64_t* n_groups) {
  if (n < 3) { set_error("%s: need offsets, target and at least one feature", sym); return 1; }
  const pdsb_column& oc = im.cols[0];
  if (oc.dtype != PDSB_I64 || oc.n_chunks != 1 || oc.null_count > 0) { set_error("%s: offsets must be one non-null Int64 chunk", sym); return 1; }
  *offs = (const int64_t*)oc.chunks[0].data + oc.chunks[0].offset;
  *n_groups = oc.chunks[0].length - 1;
  return 0;
}

// pl_lr_by / pl_lr_pred_by: inputs [offsets (Int64), y, features...]; pred selects the per-row {pred, resid} twin
void run_by(SeriesExport* in, size_t n, const uint8_t* kwp, size_t kwn, SeriesExport* ret, bool f32, bool pred) {
  run_expr(in, n, kwp, kwn, ret, REQ_LR,
    [&](const Imported& im, const Kwargs& kw, pdsb_host_result* r) {
      const int64_t* offs = nullptr;
      int64_t n_groups = 0;
      if (group_offsets(im, n, "pl_lr_by", &offs, &n_groups)) return 1;
      if (pred) return pdsb_host_grouped_lin_reg_pred(im.cols.data() + 1, (int)n - 1, offs, n_groups, &kw.k, f32, r);
      return pdsb_host_grouped_lin_reg(im.cols.data() + 1, (int)n - 1, offs, n_groups, &kw.k, f32, r);
    },
    [&](const Imported&, const Kwargs&, const pdsb_host_result& r) {
      if (!pred) return list_node("coeffs", f32, r.coeffs, r.n_rows, r.n_coef, r.valid, false);
      auto root = struct_node("", r.n_rows);
      root->children.push_back(prim_node("pred", f32, r.pred, r.n_rows, r.valid, false));
      root->children.push_back(prim_node("resid", f32, r.resid, r.n_rows, r.valid, false));
      return root;
    });
}

// pl_logistic_by / pl_logistic_pred_by: inputs [offsets (Int64), y, features...], LRKwargs; pl_logistic_coeffs's
// List<Float64> per group, or pl_logistic_pred's Float64 per row
void run_logistic_by(SeriesExport* in, size_t n, const uint8_t* kwp, size_t kwn, SeriesExport* ret, bool pred) {
  run_expr(in, n, kwp, kwn, ret, REQ_LR,
    [&](const Imported& im, const Kwargs& kw, pdsb_host_result* r) {
      const int64_t* offs = nullptr;
      int64_t n_groups = 0;
      if (group_offsets(im, n, pred ? "pl_logistic_pred_by" : "pl_logistic_by", &offs, &n_groups)) return 1;
      return pdsb_host_grouped_logistic(im.cols.data() + 1, (int)n - 1, offs, n_groups, &kw.k, pred, r);
    },
    [&](const Imported&, const Kwargs&, const pdsb_host_result& r) {
      if (!pred) return list_node("coeffs", false, r.coeffs, r.n_rows, r.n_coef, nullptr, false);
      return prim_node("pred", false, r.pred, r.n_rows, r.valid, false);
    });
}

// pl_singular_values (mode 0), pl_pca (1), pl_principal_components (2) (num_ext/pca.rs:39-182): no kwargs; mode 2 takes
// pl.lit(k, dtype=pl.UInt32) as input 0.  Float64 results whatever the input dtype.
void run_pca(SeriesExport* in, size_t n, const uint8_t* kwp, size_t kwn, SeriesExport* ret, int mode) {
  run_expr(in, n, kwp, kwn, ret, nullptr,
    [&](const Imported& im, const Kwargs&, pdsb_host_result* r) {
      int k = 0;
      size_t f0 = 0;
      if (mode == 2) {
        if (n < 2) { set_error("principal_components: need k and at least one feature"); return 1; }
        const pdsb_column& kc = im.cols[0];
        if (kc.dtype != PDSB_U32) { set_error("invalid series dtype: expected `UInt32` for k"); return 1; }
        const pdsb_chunk* ch = nullptr;
        for (int c = 0; c < kc.n_chunks && !ch; ++c) if (kc.chunks[c].length > 0) ch = &kc.chunks[c];
        if (!ch || (ch->validity && !((ch->validity[ch->offset >> 3] >> (ch->offset & 7)) & 1))) {
          set_error("principal_components: k is null"); return 1;
        }
        k = (int)std::min<uint32_t>(((const uint32_t*)ch->data)[ch->offset], 0x7fffffffu);
        f0 = 1;
      }
      return pdsb_host_pca(im.cols.data() + f0, (int)(n - f0), mode, k, r);
    },
    [&](const Imported&, const Kwargs&, const pdsb_host_result& r) {
      if (mode == 0) return list_node("singular_values", false, r.singular_values, 1, r.n_rows, nullptr, false);
      if (mode == 1) {
        auto root = struct_node("pca", r.n_rows);
        root->children.push_back(prim_node("singular_value", false, r.singular_values, r.n_rows, nullptr, false));
        root->children.push_back(list_node("weight_vector", false, r.coeffs, r.n_rows, r.n_coef, nullptr, false));
        return root;
      }
      auto root = struct_node("principal_components", r.n_rows);
      for (int j = 0; j < r.n_targets; ++j) {
        const std::string name = "pc" + std::to_string(j + 1);
        root->children.push_back(prim_node(name.c_str(), false, (const double*)r.pred + (size_t)j * r.n_rows, r.n_rows, nullptr, false));
      }
      return root;
    });
}

// pl_smooth_spline (num_ext/splines.rs:99-119): inputs x, y; kwargs {"lambda"}; a Float64 column of the input's length
void run_spline(SeriesExport* in, size_t n, const uint8_t* kwp, size_t kwn, SeriesExport* ret) {
  run_expr(in, n, kwp, kwn, ret, REQ_SPLINE,
    [&](const Imported& im, const Kwargs& kw, pdsb_host_result* r) {
      return pdsb_host_smooth_spline(im.cols.data(), (int)n, kw.k.lambda, r);
    },
    [&](const Imported& im, const Kwargs&, const pdsb_host_result& r) {
      return prim_node(im.names[0].c_str(), false, r.pred, r.n_rows, nullptr, false);
    });
}

// pl_isotonic_regression (num_ext/isotonic_regression.rs): inputs y (, w); kwargs {"has_weights", "increasing"}; a
// Float64 column of the input's length
void run_isotonic(SeriesExport* in, size_t n, const uint8_t* kwp, size_t kwn, SeriesExport* ret) {
  run_expr(in, n, kwp, kwn, ret, REQ_ISO,
    [&](const Imported& im, const Kwargs& kw, pdsb_host_result* r) {
      return pdsb_host_isotonic_regression(im.cols.data(), (int)n, kw.integer("has_weights", 0) != 0,
                                           kw.integer("increasing", 1) != 0, r);
    },
    [&](const Imported& im, const Kwargs&, const pdsb_host_result& r) {
      return prim_node(im.names[0].c_str(), false, r.pred, r.n_rows, r.valid, false);
    });
}

}  // namespace

extern "C" {

uint32_t _polars_plugin_get_version(void) { return (0u << 16) | 1u; }
int64_t pdsb_plugin_live_results(void) { return g_live_results.load(); }
const char* _polars_plugin_get_last_error_message(void) { return get_error(); }

#define DEF_EXPR(name, body, fieldbody)                                                                         \
  void _polars_plugin_##name(SeriesExport* inputs, size_t n_inputs, const uint8_t* kwargs, size_t kwargs_len,   \
                             SeriesExport* ret, void* ctx) {                                                    \
    (void)ctx;                                                                                                  \
    try { body; }                                                                                               \
    catch (const std::exception& e) { set_error("plugin error: %s", e.what()); }   /* never unwind into Polars */ \
    catch (...) { set_error("plugin error: unknown exception"); } }                                              \
  void _polars_plugin_field_##name(struct ArrowSchema* in_fields, size_t n, struct ArrowSchema* out) {          \
    (void)in_fields; (void)n; fieldbody; }

#define FIELD_COEFF(f32) { auto nd = schema_list("coeffs", f32); field_out(out, *nd); }
#define FIELD_PRED(f32) { auto nd = struct_node("pred", 0); nd->children.push_back(schema_prim("pred", f32)); nd->children.push_back(schema_prim("resid", f32)); field_out(out, *nd); }
#define FIELD_CP(f32) { auto nd = struct_node("", 0); nd->children.push_back(schema_list("coeffs", f32)); nd->children.push_back(schema_prim("pred", f32)); field_out(out, *nd); }
#define FIELD_CSV(f32) { auto nd = struct_node("", 0); nd->children.push_back(schema_list("coeffs", f32)); nd->children.push_back(schema_list("singular_values", f32)); field_out(out, *nd); }
#define FIELD_REPORT(f32) { auto nd = struct_node("lin_reg_report", 0); { auto u = std::make_unique<Node>(); u->format = "U"; u->name = "features"; nd->children.push_back(std::move(u)); } \
    const char* cn[8] = {"beta", "std_err", "t", "p>|t|", "0.025", "0.975", "r2", "adj_r2"};                     \
    for (int c = 0; c < 8; ++c) nd->children.push_back(schema_prim(cn[c], f32)); field_out(out, *nd); }

// output_type_func of each symbol mirrors the reference, including the knowingly-wrong multi-target ones
// (linear_regression.rs:515-517, 586-587)
DEF_EXPR(pl_lr,               run_lr(inputs, n_inputs, kwargs, kwargs_len, ret, false, false, false), FIELD_COEFF(false))
DEF_EXPR(pl_lr_pred,          run_lr(inputs, n_inputs, kwargs, kwargs_len, ret, false, true, false),  FIELD_PRED(false))
DEF_EXPR(pl_lr_w_rcond,       run_lr(inputs, n_inputs, kwargs, kwargs_len, ret, false, false, true),  FIELD_CSV(false))
DEF_EXPR(pl_lr_multi,         run_multi(inputs, n_inputs, kwargs, kwargs_len, ret, false, false),     FIELD_COEFF(false))
DEF_EXPR(pl_lr_multi_pred,    run_multi(inputs, n_inputs, kwargs, kwargs_len, ret, false, true),      FIELD_PRED(false))
DEF_EXPR(pl_lin_reg_report,   run_report(inputs, n_inputs, kwargs, kwargs_len, ret, false, false),    FIELD_REPORT(false))
DEF_EXPR(pl_wls_report,       run_report(inputs, n_inputs, kwargs, kwargs_len, ret, false, true),     FIELD_REPORT(false))
DEF_EXPR(pl_recursive_lr,     run_online(inputs, n_inputs, kwargs, kwargs_len, ret, false, false),    FIELD_CP(false))
DEF_EXPR(pl_rolling_lr,       run_online(inputs, n_inputs, kwargs, kwargs_len, ret, false, true),     FIELD_CP(false))
DEF_EXPR(pl_lr_by,            run_by(inputs, n_inputs, kwargs, kwargs_len, ret, false, false),        FIELD_COEFF(false))
DEF_EXPR(pl_logistic_coeffs,  run_logistic(inputs, n_inputs, kwargs, kwargs_len, ret, false),         FIELD_COEFF(false))
DEF_EXPR(pl_logistic_pred,    run_logistic(inputs, n_inputs, kwargs, kwargs_len, ret, true),          { auto nd = schema_prim("pred", false); field_out(out, *nd); })

// num_ext/pca.rs:10-37.  The principal_components twin declares pc1..pc{number of inputs}: the inputs include the k
// literal, so one field more than there are features (the reference's declaration, kept)
DEF_EXPR(pl_singular_values,      run_pca(inputs, n_inputs, kwargs, kwargs_len, ret, 0), { auto nd = schema_list("singular_values", false); field_out(out, *nd); })
DEF_EXPR(pl_pca,                  run_pca(inputs, n_inputs, kwargs, kwargs_len, ret, 1),
         { auto nd = struct_node("pca", 0); nd->children.push_back(schema_prim("singular_value", false));
           nd->children.push_back(schema_list("weight_vector", false)); field_out(out, *nd); })
DEF_EXPR(pl_principal_components, run_pca(inputs, n_inputs, kwargs, kwargs_len, ret, 2),
         { auto nd = struct_node("principal_components", 0);
           for (size_t i = 0; i < n; ++i) nd->children.push_back(schema_prim(("pc" + std::to_string(i + 1)).c_str(), false));
           field_out(out, *nd); })

// num_ext/splines.rs:99 (#[polars_expr(output_type=Float64)])
// (#[polars_expr(output_type=Float64)]: Float64 under the first input's name)
DEF_EXPR(pl_smooth_spline,        run_spline(inputs, n_inputs, kwargs, kwargs_len, ret),
         { auto nd = schema_prim(n > 0 && in_fields[0].name ? in_fields[0].name : "", false); field_out(out, *nd); })

// num_ext/isotonic_regression.rs (#[polars_expr(output_type=Float64)]: Float64 under the first input's name)
DEF_EXPR(pl_isotonic_regression,  run_isotonic(inputs, n_inputs, kwargs, kwargs_len, ret),
         { auto nd = schema_prim(n > 0 && in_fields[0].name ? in_fields[0].name : "", false); field_out(out, *nd); })

DEF_EXPR(pl_lr_f32,            run_lr(inputs, n_inputs, kwargs, kwargs_len, ret, true, false, false), FIELD_COEFF(true))
DEF_EXPR(pl_lr_pred_f32,        run_lr(inputs, n_inputs, kwargs, kwargs_len, ret, true, true, false),  FIELD_PRED(true))
DEF_EXPR(pl_lr_w_rcond_f32,     run_lr(inputs, n_inputs, kwargs, kwargs_len, ret, true, false, true),  FIELD_CSV(true))
DEF_EXPR(pl_lr_multi_f32,       run_multi(inputs, n_inputs, kwargs, kwargs_len, ret, true, false),     FIELD_COEFF(true))
DEF_EXPR(pl_lr_multi_pred_f32,  run_multi(inputs, n_inputs, kwargs, kwargs_len, ret, true, true),      FIELD_PRED(true))
DEF_EXPR(pl_lin_reg_report_f32, run_report(inputs, n_inputs, kwargs, kwargs_len, ret, true, false),    FIELD_REPORT(true))
DEF_EXPR(pl_wls_report_f32,     run_report(inputs, n_inputs, kwargs, kwargs_len, ret, true, true),     FIELD_REPORT(true))
DEF_EXPR(pl_recursive_lr_f32,   run_online(inputs, n_inputs, kwargs, kwargs_len, ret, true, false),    FIELD_CP(true))
DEF_EXPR(pl_rolling_lr_f32,     run_online(inputs, n_inputs, kwargs, kwargs_len, ret, true, true),     FIELD_CP(true))
DEF_EXPR(pl_lr_by_f32,          run_by(inputs, n_inputs, kwargs, kwargs_len, ret, true, false),        FIELD_COEFF(true))

// polars_plugin_group_abi.h: lin_reg(return_pred=True).over(key) in one call; pl_lr_pred's output type
DEF_EXPR(pl_lr_pred_by,         run_by(inputs, n_inputs, kwargs, kwargs_len, ret, false, true),        FIELD_PRED(false))
DEF_EXPR(pl_lr_pred_by_f32,     run_by(inputs, n_inputs, kwargs, kwargs_len, ret, true, true),         FIELD_PRED(true))

// polars_plugin_group_logistic_abi.h: group_by().agg(logistic_reg) and logistic_reg(return_pred=True).over(key) in one
// call; pl_logistic_coeffs's and pl_logistic_pred's output types
DEF_EXPR(pl_logistic_by,        run_logistic_by(inputs, n_inputs, kwargs, kwargs_len, ret, false),    FIELD_COEFF(false))
DEF_EXPR(pl_logistic_pred_by,   run_logistic_by(inputs, n_inputs, kwargs, kwargs_len, ret, true),
         { auto nd = schema_prim("pred", false); field_out(out, *nd); })

}  // extern "C"
