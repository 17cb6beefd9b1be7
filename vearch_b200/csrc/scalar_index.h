// Scalar index of one indexed table field, kept in HBM (table/scalar_index_manager.cc: one index per field).  Numeric
// fields keep a native-width value column with a validity bit per document; STRING fields an int32 dictionary code per
// document; STRINGARRAY fields an (offset, count) run per document into an append-only pool of codes.  The term -> code
// dictionary stays on the host.  New and changed values are staged on the host and reach the device in batches
// (flush); filters are evaluated on the device columns (kernels_filter.cu).
#pragma once
#include <stdint.h>

#include <string>
#include <unordered_map>
#include <vector>

#include "kernels.h"

namespace gb {

// width in bytes of a numeric field's raw little-endian value, 0 for the string types
int scalar_width(int data_type);

class ScalarColumn {
 public:
  ScalarColumn() = default;
  ScalarColumn(const ScalarColumn&) = delete;
  ScalarColumn& operator=(const ScalarColumn&) = delete;
  ScalarColumn(ScalarColumn&& o) noexcept { *this = std::move(o); }
  ScalarColumn& operator=(ScalarColumn&& o) noexcept;
  ~ScalarColumn() { release(); }

  bool built() const { return built_; }
  // Mutators: the caller holds the table exclusively and has made the column's device current.
  // The columns of documents [0, values.size()) in one upload; drops whatever was staged.  0, or -1 (last_error)
  int build(int data_type, const std::vector<std::string>& values);
  void release();  // frees the device columns and the dictionary; the field is no longer indexed
  // document docid now holds `value`; `old`: its previous value (nullptr for a new document)
  void stage(int docid, const std::string& value, const std::string* old);
  int64_t staged() const { return (int64_t)st_doc_.size(); }
  // applies the staged values, in staging order per document, on st and waits for them.  0, or -1 (last_error)
  int flush(cudaStream_t st);
  // more than half of the string-array pool belongs to replaced values: build() again re-packs it
  bool wants_repack() const { return dt_is_array() && pool_dead_ * 2 > pool_size_; }

  // Readers (table held shared).  Fills d's column fields; kind, width and ncol included.
  void describe(FilterDesc* d) const;
  // sorted distinct codes of the terms the dictionary knows (the others match no document)
  void codes_of(const std::vector<std::string>& terms, std::vector<int32_t>* out) const;
  int data_type() const { return dt_; }
  int64_t mem_bytes() const;  // device columns, pool and dictionary

 private:
  bool dt_is_array() const;
  int32_t code_for(const std::string& term);  // the term's code, added to the dictionary when new
  int grow(int64_t docs, cudaStream_t st);     // device columns hold at least `docs` documents
  int grow_pool(int64_t codes, cudaStream_t st);

  bool built_ = false;
  int dt_ = 0, width_ = 0;
  int64_t cap_ = 0;   // documents the device columns can hold
  int64_t ndoc_ = 0;  // documents written on the device: [0, ndoc_)
  void* col_ = nullptr;          // numeric values, width_ bytes each
  uint32_t* valid_ = nullptr;    // numeric validity bits
  int32_t* codes_ = nullptr;     // STRING codes
  int64_t* arr_off_ = nullptr;   // STRINGARRAY runs
  int32_t* arr_cnt_ = nullptr;
  int32_t* pool_ = nullptr;
  int64_t pool_size_ = 0, pool_cap_ = 0, pool_dead_ = 0;
  std::unordered_map<std::string, int32_t> dict_;
  int64_t dict_bytes_ = 0;
  // staged: document, raw value (numeric: the value's bytes; STRING: code; STRINGARRAY: element count), numeric
  // validity; STRINGARRAY element codes in st_pool_, in staging order
  std::vector<int32_t> st_doc_;
  std::vector<uint64_t> st_val_;
  std::vector<uint8_t> st_ok_;
  std::vector<int32_t> st_pool_;
};

}  // namespace gb
