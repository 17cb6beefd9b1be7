// ScalarColumn (see scalar_index.h): device columns of an indexed scalar field, built in bulk or fed in staged batches.
#include "scalar_index.h"

#include <string.h>

#include <algorithm>
#include <numeric>

#include "engine.h"
#include "mem_ledger.h"

namespace gb {

int scalar_width(int dt) {
  switch (dt) {
    case DT_INT:
    case DT_FLOAT: return 4;
    case DT_BOOL: return 1;
    case DT_LONG:
    case DT_DOUBLE:
    case DT_DATE: return 8;
    default: return 0;
  }
}

namespace {
constexpr int64_t kMinColumnDocs = 8192;

int64_t count001(const std::string& s) { return 1 + (int64_t)std::count(s.begin(), s.end(), '\001'); }

template <typename F>
void for_each001(const std::string& s, F&& f) {  // the \001-separated items, an empty one included
  size_t a = 0;
  while (true) {
    const size_t b = s.find('\001', a);
    f(s.substr(a, b == std::string::npos ? std::string::npos : b - a));
    if (b == std::string::npos) break;
    a = b + 1;
  }
}

// the raw value of a numeric field as the column stores it; false: wrong width, the document has no valid value
bool raw_value(int width, const std::string& v, uint64_t* raw) {
  *raw = 0;
  if (width == 0 || v.size() != (size_t)width) return false;
  memcpy(raw, v.data(), (size_t)width);
  return true;
}

template <typename T>
cudaError_t dev_alloc(T** p, int64_t n) {
  *p = nullptr;
  return n > 0 ? mem::dev_malloc(p, (size_t)n * sizeof(T)) : cudaSuccess;
}
// a zeroed buffer of n elements holding the first `keep` elements of old (old is freed)
template <typename T>
cudaError_t dev_regrow(T** p, int64_t keep, int64_t n, cudaStream_t st) {
  T* q = nullptr;
  cudaError_t e = dev_alloc(&q, n);
  if (e == cudaSuccess) e = cudaMemsetAsync(q, 0, (size_t)n * sizeof(T), st);
  if (e == cudaSuccess && keep > 0) e = cudaMemcpyAsync(q, *p, (size_t)keep * sizeof(T), cudaMemcpyDeviceToDevice, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) {
    mem::dev_free(q);
    return e;
  }
  mem::dev_free(*p);
  *p = q;
  return cudaSuccess;
}
}  // namespace

ScalarColumn& ScalarColumn::operator=(ScalarColumn&& o) noexcept {
  if (this == &o) return *this;
  release();
  built_ = o.built_, dt_ = o.dt_, width_ = o.width_, cap_ = o.cap_, ndoc_ = o.ndoc_;
  col_ = o.col_, valid_ = o.valid_, codes_ = o.codes_, arr_off_ = o.arr_off_, arr_cnt_ = o.arr_cnt_, pool_ = o.pool_;
  pool_size_ = o.pool_size_, pool_cap_ = o.pool_cap_, pool_dead_ = o.pool_dead_;
  dict_ = std::move(o.dict_);
  dict_bytes_ = o.dict_bytes_;
  st_doc_ = std::move(o.st_doc_), st_val_ = std::move(o.st_val_), st_ok_ = std::move(o.st_ok_);
  st_pool_ = std::move(o.st_pool_);
  o.col_ = nullptr, o.valid_ = nullptr, o.codes_ = nullptr, o.arr_off_ = nullptr, o.arr_cnt_ = nullptr, o.pool_ = nullptr;
  o.built_ = false, o.cap_ = o.ndoc_ = o.pool_size_ = o.pool_cap_ = o.pool_dead_ = o.dict_bytes_ = 0;
  return *this;
}

bool ScalarColumn::dt_is_array() const { return dt_ == DT_STRINGARRAY; }

void ScalarColumn::release() {
  for (void* p : {col_, (void*)valid_, (void*)codes_, (void*)arr_off_, (void*)arr_cnt_, (void*)pool_})
    mem::dev_free(p);
  col_ = nullptr, valid_ = nullptr, codes_ = nullptr, arr_off_ = nullptr, arr_cnt_ = nullptr, pool_ = nullptr;
  built_ = false;
  cap_ = ndoc_ = pool_size_ = pool_cap_ = pool_dead_ = dict_bytes_ = 0;
  dict_ = {};
  st_doc_ = {}, st_val_ = {}, st_ok_ = {}, st_pool_ = {};
}

int32_t ScalarColumn::code_for(const std::string& term) {
  auto r = dict_.emplace(term, (int32_t)dict_.size());
  if (r.second) dict_bytes_ += (int64_t)(term.size() + sizeof(std::string) + sizeof(int32_t) + 2 * sizeof(void*));
  return r.first->second;
}

int ScalarColumn::grow(int64_t docs, cudaStream_t st) {
  if (docs <= cap_) return 0;
  int64_t cap = std::max(std::max(docs, 2 * cap_), kMinColumnDocs);
  cap = (cap + 31) / 32 * 32;
  if (width_) {
    uint8_t* c = static_cast<uint8_t*>(col_);
    GB_CUDA(dev_regrow(&c, cap_ * width_, cap * width_, st));
    col_ = c;
    GB_CUDA(dev_regrow(&valid_, cap_ / 32, cap / 32, st));
  } else if (dt_is_array()) {
    GB_CUDA(dev_regrow(&arr_off_, cap_, cap, st));
    GB_CUDA(dev_regrow(&arr_cnt_, cap_, cap, st));
  } else {
    GB_CUDA(dev_regrow(&codes_, cap_, cap, st));
  }
  cap_ = cap;
  return 0;
}

int ScalarColumn::grow_pool(int64_t codes, cudaStream_t st) {
  if (codes <= pool_cap_) return 0;
  const int64_t cap = std::max(std::max(codes, 2 * pool_cap_), kMinColumnDocs);
  GB_CUDA(dev_regrow(&pool_, pool_size_, cap, st));
  pool_cap_ = cap;
  return 0;
}

int ScalarColumn::build(int data_type, const std::vector<std::string>& values) {
  std::unordered_map<std::string, int32_t> dict = std::move(dict_);
  const int64_t dict_bytes = dict_bytes_;
  release();  // the dictionary survives a re-build: codes stay what they were
  dict_ = std::move(dict);
  dict_bytes_ = dict_bytes;
  dt_ = data_type;
  width_ = scalar_width(dt_);
  built_ = true;
  const int64_t n = (int64_t)values.size();
  cudaStream_t st = cudaStreamPerThread;
  if (grow(n, st)) return -1;
  if (width_) {
    std::vector<uint8_t> col((size_t)n * width_, 0);
    std::vector<uint32_t> valid((size_t)(n + 31) / 32, 0);
    for (int64_t d = 0; d < n; d++) {
      uint64_t raw;
      if (!raw_value(width_, values[d], &raw)) continue;
      memcpy(col.data() + d * width_, &raw, (size_t)width_);
      valid[d >> 5] |= 1u << (d & 31);
    }
    GB_CUDA(cudaMemcpyAsync(col_, col.data(), col.size(), cudaMemcpyHostToDevice, st));
    GB_CUDA(cudaMemcpyAsync(valid_, valid.data(), valid.size() * 4, cudaMemcpyHostToDevice, st));
  } else if (dt_is_array()) {
    std::vector<int64_t> off((size_t)n);
    std::vector<int32_t> cnt((size_t)n), pool;
    for (int64_t d = 0; d < n; d++) {
      off[d] = (int64_t)pool.size();
      for_each001(values[d], [&](const std::string& e) { pool.push_back(code_for(e)); });
      cnt[d] = (int32_t)((int64_t)pool.size() - off[d]);
    }
    if (grow_pool((int64_t)pool.size(), st)) return -1;
    GB_CUDA(cudaMemcpyAsync(arr_off_, off.data(), off.size() * 8, cudaMemcpyHostToDevice, st));
    GB_CUDA(cudaMemcpyAsync(arr_cnt_, cnt.data(), cnt.size() * 4, cudaMemcpyHostToDevice, st));
    GB_CUDA(cudaMemcpyAsync(pool_, pool.data(), pool.size() * 4, cudaMemcpyHostToDevice, st));
    pool_size_ = (int64_t)pool.size();
  } else {
    std::vector<int32_t> codes((size_t)n);
    for (int64_t d = 0; d < n; d++) codes[d] = code_for(values[d]);
    GB_CUDA(cudaMemcpyAsync(codes_, codes.data(), codes.size() * 4, cudaMemcpyHostToDevice, st));
  }
  GB_CUDA(cudaStreamSynchronize(st));
  ndoc_ = n;
  return 0;
}

void ScalarColumn::stage(int docid, const std::string& value, const std::string* old) {
  st_doc_.push_back(docid);
  if (width_) {
    uint64_t raw;
    st_ok_.push_back(raw_value(width_, value, &raw) ? 1 : 0);
    st_val_.push_back(raw);
  } else if (dt_is_array()) {
    const size_t before = st_pool_.size();
    for_each001(value, [&](const std::string& e) { st_pool_.push_back(code_for(e)); });
    st_val_.push_back(st_pool_.size() - before);
    if (old) pool_dead_ += count001(*old);  // its run stays in the pool, unreferenced
  } else {
    st_val_.push_back((uint64_t)(uint32_t)code_for(value));
  }
}

int ScalarColumn::flush(cudaStream_t st) {
  const int64_t m = staged();
  if (m == 0) return 0;
  // the last staging of each document wins; runs of string-array codes start where their staging put them
  std::vector<int64_t> start;
  if (dt_is_array()) {
    start.resize((size_t)m);
    int64_t a = 0;
    for (int64_t i = 0; i < m; i++) start[i] = a, a += (int64_t)st_val_[i];
  }
  std::vector<int64_t> order((size_t)m);
  std::iota(order.begin(), order.end(), 0);
  std::stable_sort(order.begin(), order.end(), [&](int64_t a, int64_t b) { return st_doc_[a] < st_doc_[b]; });
  std::vector<int32_t> docs;
  std::vector<uint64_t> vals, offs;
  std::vector<uint8_t> ok;
  docs.reserve((size_t)m);
  for (int64_t j = 0; j < m; j++) {
    const int64_t i = order[j];
    if (j + 1 < m && st_doc_[order[j + 1]] == st_doc_[i]) continue;
    docs.push_back(st_doc_[i]);
    vals.push_back(st_val_[i]);
    if (width_) ok.push_back(st_ok_[i]);
    if (dt_is_array()) offs.push_back((uint64_t)(pool_size_ + start[i]));
  }
  const int64_t mk = (int64_t)docs.size();
  if (grow((int64_t)docs.back() + 1, st)) return -1;
  if (dt_is_array() && grow_pool(pool_size_ + (int64_t)st_pool_.size(), st)) return -1;
  Scratch s(st);
  int32_t* ddocs = s.alloc_n<int32_t>((size_t)mk);
  uint64_t* dvals = s.alloc_n<uint64_t>((size_t)mk * 2);
  uint8_t* dok = s.alloc_n<uint8_t>((size_t)mk);
  if (!ddocs || !dvals || !dok) return -1;
  GB_CUDA(cudaMemcpyAsync(ddocs, docs.data(), (size_t)mk * 4, cudaMemcpyHostToDevice, st));
  GB_CUDA(cudaMemcpyAsync(dvals, vals.data(), (size_t)mk * 8, cudaMemcpyHostToDevice, st));
  if (width_) {
    GB_CUDA(cudaMemcpyAsync(dok, ok.data(), (size_t)mk, cudaMemcpyHostToDevice, st));
    GB_CUDA(launch_scatter_column(ddocs, dvals, dok, mk, width_, col_, valid_, st));
  } else if (dt_is_array()) {
    GB_CUDA(cudaMemcpyAsync(dvals + mk, offs.data(), (size_t)mk * 8, cudaMemcpyHostToDevice, st));
    if (!st_pool_.empty())
      GB_CUDA(cudaMemcpyAsync(pool_ + pool_size_, st_pool_.data(), st_pool_.size() * 4, cudaMemcpyHostToDevice, st));
    GB_CUDA(launch_scatter_column(ddocs, dvals + mk, nullptr, mk, 8, arr_off_, nullptr, st));
    GB_CUDA(launch_scatter_column(ddocs, dvals, nullptr, mk, 4, arr_cnt_, nullptr, st));
  } else {
    GB_CUDA(launch_scatter_column(ddocs, dvals, nullptr, mk, 4, codes_, nullptr, st));
  }
  GB_CUDA(cudaStreamSynchronize(st));
  if (dt_is_array()) pool_size_ += (int64_t)st_pool_.size();
  ndoc_ = std::max<int64_t>(ndoc_, (int64_t)docs.back() + 1);
  st_doc_.clear(), st_val_.clear(), st_ok_.clear(), st_pool_.clear();
  return 0;
}

void ScalarColumn::describe(FilterDesc* d) const {
  d->kind = width_ ? kFilterNumeric : (dt_is_array() ? kFilterStringArray : kFilterString);
  d->width = width_;
  d->is_float = dt_ == DT_FLOAT || dt_ == DT_DOUBLE;
  d->ncol = ndoc_;
  d->col = col_;
  d->valid = valid_;
  d->codes = codes_;
  d->arr_off = arr_off_;
  d->arr_cnt = arr_cnt_;
  d->pool = pool_;
}

void ScalarColumn::codes_of(const std::vector<std::string>& terms, std::vector<int32_t>* out) const {
  out->clear();
  for (const auto& t : terms) {
    auto it = dict_.find(t);
    if (it != dict_.end()) out->push_back(it->second);
  }
  std::sort(out->begin(), out->end());
  out->erase(std::unique(out->begin(), out->end()), out->end());
}

int64_t ScalarColumn::mem_bytes() const {
  int64_t b = dict_bytes_;
  if (width_) b += cap_ * width_ + cap_ / 8;
  else if (dt_is_array()) b += cap_ * 12 + pool_cap_ * 4;
  else b += cap_ * 4;
  return b;
}

}  // namespace gb
