// SURVEY 8f N-1: gamma's on-disk index files, byte for byte, so a partition dumped by the CPU engine
// loads into this one without retraining (and the other way round).
//
// Layout (little endian; faiss "fourcc" = the four characters in file order), restated from
//   GammaIVFFlatIndex::Dump / Load   index/impl/gamma_index_ivfflat.cc:807-892   <dir>/<name>/ivfflat.index
//   GammaIVFPQIndex::Dump / Load     index/impl/gamma_index_ivfpq.cc:1019-1116   <dir>/<name>/ivfpq.index
//   write_ivf_header, write_index_header, write_direct_map, write_product_quantizer,
//   WriteInvertedLists / ReadInvertedLists                                      index/index_io.cc:15-194
//   faiss::write_index(IndexFlat) (faiss v1.14.1 impl/index_write.cpp; not vendored: restated)
//
//   u32  "IvFl" | "IwPQ"
//   ivf header : index header { i32 d, i64 ntotal, i64 1<<20, i64 1<<20, u8 is_trained, i32 metric (0 = IP, 1 = L2) }
//                u64 nlist, u64 nprobe,
//                quantizer = u32 "IxF2" | "IxFI", index header (ntotal = nlist), u64 nlist*d, nlist*d fp32
//                direct map = u8 type (0 = none), u64 0
//   IwPQ only  : u8 by_residual, u64 code_size, u64 d, u64 M, u64 nbits, u64 M*ksub*dsub, fp32 centroids [M][ksub][dsub]
//                (ksub = 2^nbits, code_size = ceil(M nbits / 8): the list codes bit-packed as faiss PQEncoderGeneric)
//   lists      : u32 "ilar", u64 nlist, u64 code_bytes, u32 "full", u64 nlist, u64 sizes[nlist],
//                per non-empty list: codes[size * code_bytes], i64 ids[size] (top bit = tombstone)
//   IvFl only  : i32 indexed_count
// An IndexHNSWFlat coarse quantiser ("IHNf") is read for its centroids (the graph is skipped: the coarse
// search here is exact); Dump always writes the IndexFlat form.  An OPQ block ("LTra") follows the product quantizer when the table has opq.
//
// The quantised types the reference writes no file of that this engine could read (IVFPQFastScan, VEARCH, BINARYIVF:
// none; IVFRABITQ: faiss's IndexIVFRaBitQ) get files of this engine's own, under names the reference never opens, so a
// CPU partition never meets them and a CPU-written ivfrabitq.index is never read here.  They share the skeleton above,
// the IvFl trailing i32 indexed_count included, with their own fourcc and codec block after the direct map:
//   "GbFS" gb_ivfpqfs.index   : u64 code_size, u64 d, u64 M, u64 nbits (4), u64 M*16*dsub, fp32 codebook [M][16][dsub]
//   "GbRQ" gb_ivfrabitq.index : u64 code_size, i32 nb_bits, i32 qb
//   "GbVR" gb_vearch.index    : u64 code_size, i32 nsubvector, i32 nblocks, f64 ns_threshold (NaN: none), u8 reordering,
//                               u64 16*d, fp32 block codebooks [16 d] (each block's centres in their trained order)
//   "GbBI" gb_binaryivf.index : u64 code_size (d / 8), u64 nlist*code_size, packed centroids [nlist][d / 8]
// An index with SOAR spilling (soar_lambda > 0, DESIGN.md §8) writes the same file under the variant fourcc "GsFS" /
// "GsRQ" / "GsVR" (for "GbFS" / "GbRQ" / "GbVR") with f64 soar_lambda right after the codec block; its lists hold both
// entries of every spilled row, two live entries per vid in two different lists.
// d is in bits for BINARYIVF, whose coarse-quantiser block holds the float k-means centroids (metric L2).  A file is
// refused unless d, nlist, metric and every codec parameter match the table; the index is then left untrained.
#include <errno.h>
#include <math.h>
#include <stdio.h>
#include <string.h>
#include <sys/stat.h>

#include <algorithm>
#include <functional>
#include <memory>

#include "common.cuh"
#include "index.h"

namespace gb {

namespace {

struct FileCloser {
  void operator()(FILE* f) const {
    if (f) fclose(f);
  }
};
using FilePtr = std::unique_ptr<FILE, FileCloser>;

constexpr uint32_t fourcc(const char (&s)[5]) {
  return (uint32_t)(uint8_t)s[0] | (uint32_t)(uint8_t)s[1] << 8 | (uint32_t)(uint8_t)s[2] << 16 |
         (uint32_t)(uint8_t)s[3] << 24;
}

template <class T>
bool wr(FILE* f, const T& v) {
  return fwrite(&v, sizeof(T), 1, f) == 1;
}
template <class T>
bool rd(FILE* f, T* v) {
  return fread(v, sizeof(T), 1, f) == 1;
}
bool wr_bytes(FILE* f, const void* p, size_t n) { return n == 0 || fwrite(p, 1, n, f) == n; }
bool rd_bytes(FILE* f, void* p, size_t n) { return n == 0 || fread(p, 1, n, f) == n; }

// write_index_header (index_io.cc:15-23)
bool wr_index_header(FILE* f, int d, int64_t ntotal, int metric) {
  const int64_t dummy = 1 << 20;
  const uint8_t trained = 1;
  const int32_t mt = metric == kMetricL2 ? 1 : 0;  // faiss::METRIC_INNER_PRODUCT = 0, METRIC_L2 = 1
  return wr<int32_t>(f, d) && wr<int64_t>(f, ntotal) && wr(f, dummy) && wr(f, dummy) && wr(f, trained) && wr(f, mt);
}
struct IndexHeader {
  int32_t d = 0, metric = 0;
  int64_t ntotal = 0;
  uint8_t trained = 0;
};
bool rd_index_header(FILE* f, IndexHeader* h) {
  int64_t dummy;
  if (!(rd(f, &h->d) && rd(f, &h->ntotal) && rd(f, &dummy) && rd(f, &dummy) && rd(f, &h->trained) && rd(f, &h->metric)))
    return false;
  if (h->metric > 1) {  // faiss writes metric_arg for the exotic metrics
    float arg;
    if (!rd(f, &arg)) return false;
  }
  return true;
}

int fail(const std::string& msg) {
  set_last_error(msg);
  return -1;
}

}  // namespace

// IVF-Flat rows are padded to a multiple of 4 floats here; gamma's are not
GammaFileFormat IVFFlatIndex::gamma_format() const { return {"ivfflat.index", fourcc("IvFl"), (uint64_t)d_ * 4, true}; }
GammaFileFormat IVFPQIndex::gamma_format() const { return {"ivfpq.index", fourcc("IwPQ"), (uint64_t)code_bytes(), false}; }
// a spilled index (soar_lambda > 0) writes the variant fourcc ("Gs" for "Gb") and its lambda after the codec block
GammaFileFormat IVFPQFastScanIndex::gamma_format() const {
  return {"gb_ivfpqfs.index", spilled() ? fourcc("GsFS") : fourcc("GbFS"), (uint64_t)code_bytes(), true};
}
GammaFileFormat RaBitQIndex::gamma_format() const {
  return {"gb_ivfrabitq.index", spilled() ? fourcc("GsRQ") : fourcc("GbRQ"), (uint64_t)code_bytes(), true};
}
GammaFileFormat VearchIndex::gamma_format() const {
  return {"gb_vearch.index", spilled() ? fourcc("GsVR") : fourcc("GbVR"), (uint64_t)code_bytes(), true};
}
GammaFileFormat BinaryIvfIndex::gamma_format() const {
  return {"gb_binaryivf.index", fourcc("GbBI"), (uint64_t)code_bytes(), true};
}

// ---- Dump: capture, then write ----------------------------------------------------------------
int Index::dump_gamma(const std::string& dir, const std::string& abs_name) {
  GammaImage img;
  return capture_gamma(&img) ? -1 : write_gamma_image(img, dir, abs_name);
}

int IvfIndex::capture_gamma(GammaImage* img) {
  if (!trained_ || !gamma_format().file) return 0;  // "gamma index is not trained, skip dumping" (ivfflat.cc:808-811)
  std::lock_guard<std::mutex> bg(build_mu_);  // no list mutation while the lists are copied out
  if (capture_head(indexed_count_, img)) return -1;
  return capture_lists({this}, img);
}

int IvfIndex::capture_head(int64_t indexed, GammaImage* img) {
  const GammaFileFormat gf = gamma_format();
  cudaSetDevice(device_);
  img->file = gf.file;
  img->code_size = gf.code_size;
  img->nlist = nlist_;
  img->indexed = indexed;
  img->indexed_count = gf.indexed_count;
  std::vector<float> cent((size_t)nlist_ * d_);
  if (get_centroids(cent.data())) return -1;
  char* buf = nullptr;
  size_t len = 0;
  FILE* f = open_memstream(&buf, &len);
  if (!f) return fail("cannot capture the index header");
  bool ok = wr<uint32_t>(f, gf.magic);
  // write_ivf_header (index_io.cc:41-47)
  ok = ok && wr_index_header(f, d_, indexed, mp_.metric);
  ok = ok && wr<uint64_t>(f, (uint64_t)nlist_) && wr<uint64_t>(f, (uint64_t)mp_.nprobe);
  ok = ok && wr<uint32_t>(f, mp_.metric == kMetricL2 ? fourcc("IxF2") : fourcc("IxFI"));
  ok = ok && wr_index_header(f, d_, nlist_, mp_.metric);
  ok = ok && wr<uint64_t>(f, (uint64_t)cent.size()) && wr_bytes(f, cent.data(), cent.size() * 4);  // WRITEXBVECTOR
  ok = ok && wr<uint8_t>(f, 0) && wr<uint64_t>(f, 0);                                              // direct map: none
  ok = ok && dump_gamma_extra(f) == 0;
  if (spilled()) ok = ok && wr<double>(f, mp_.soar_lambda);
  ok = fclose(f) == 0 && ok;
  if (ok) img->head.assign(buf, len);
  free(buf);
  return ok ? 0 : fail("cannot capture the trained state of the index");
}

int IvfIndex::capture_lists(const std::vector<IvfIndex*>& shards, GammaImage* img) {
  const int S = (int)shards.size(), cb = (int)img->code_size, src_cb = shards[0]->code_bytes();
  img->parts.clear();
  img->parts.resize(S);
  std::vector<std::pair<int, std::vector<PackChunk>>> by_device;  // one launch per device
  for (int s = 0; s < S; s++) {
    const IvfLists* lists = shards[s]->lists_.get();
    GammaImage::Part& part = img->parts[s];
    part.lens = lists ? lists->lens() : std::vector<int>(img->nlist, 0);
    if (!lists || part.stage.alloc((size_t)lists->pack_bytes(cb), shards[s]->device_)) {
      if (!lists) continue;
      return -1;
    }
    auto at = std::find_if(by_device.begin(), by_device.end(), [&](const auto& e) { return e.first == shards[s]->device_; });
    if (at == by_device.end()) at = by_device.emplace(by_device.end(), shards[s]->device_, std::vector<PackChunk>());
    lists->pack_chunks(cb, part.stage.data(), &at->second);
  }
  for (auto& [dev, chunks] : by_device) {
    if (chunks.empty()) continue;
    uintptr_t bits = (uintptr_t)src_cb | (uintptr_t)cb | 16;
    for (const PackChunk& c : chunks)
      bits |= (uintptr_t)c.src_codes | (uintptr_t)c.src_ids | (uintptr_t)c.dst_codes | (uintptr_t)c.dst_ids;
    const int align = (int)(bits & (~bits + 1));  // lowest set bit: at most 16
    cudaSetDevice(dev);
    cudaStream_t st = nullptr;
    GB_CUDA(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    cudaError_t e;
    {
      Scratch sc(st);
      PackChunk* d_chunks = sc.alloc_n<PackChunk>(chunks.size());
      e = d_chunks ? cudaMemcpyAsync(d_chunks, chunks.data(), sizeof(PackChunk) * chunks.size(), cudaMemcpyHostToDevice, st)
                   : cudaErrorMemoryAllocation;
      if (e == cudaSuccess) e = launch_list_pack(d_chunks, (int)chunks.size(), src_cb, cb, align, st);
      if (e == cudaSuccess) e = cudaStreamSynchronize(st);  // the stage is complete before the lock is released
    }
    cudaStreamDestroy(st);
    if (e != cudaSuccess) return fail(std::string("list pack: ") + cudaGetErrorString(e));
  }
  return 0;
}

int write_gamma_image(const GammaImage& img, const std::string& dir, const std::string& abs_name) {
  if (img.file.empty()) return 0;
  const std::string index_dir = dir + "/" + abs_name;
  mkdir(dir.c_str(), 0755);
  if (mkdir(index_dir.c_str(), 0755) && errno != EEXIST) return fail("mkdir error, index dir=" + index_dir);
  const std::string path = index_dir + "/" + img.file;
  FilePtr fp(fopen(path.c_str(), "wb"));
  FILE* f = fp.get();
  if (!f) return fail("cannot open " + path);
  const int S = (int)img.parts.size(), nlist = img.nlist;
  const uint64_t cb = img.code_size;
  std::vector<int> lens(nlist, 0);
  for (const GammaImage::Part& p : img.parts)
    for (int l = 0; l < nlist; l++) lens[l] += p.lens[l];
  // WriteInvertedLists (index_io.cc:108-141)
  bool ok = wr_bytes(f, img.head.data(), img.head.size()) && wr<uint32_t>(f, fourcc("ilar")) &&
            wr<uint64_t>(f, (uint64_t)nlist) && wr<uint64_t>(f, cb) && wr<uint32_t>(f, fourcc("full")) &&
            wr<uint64_t>(f, (uint64_t)nlist);
  for (int l = 0; ok && l < nlist; l++) ok = wr<uint64_t>(f, (uint64_t)lens[l]);
  if (ok && S == 1) {
    ok = img.parts[0].stage.write(f, 0, img.parts[0].stage.size());
  } else if (ok) {
    std::vector<std::vector<uint8_t>> part(S);
    std::vector<size_t> at(S, 0);  // list l of shard s starts at part[s][at[s]]: its codes, then its ids
    for (int s = 0; s < S; s++) {
      part[s].resize(img.parts[s].stage.size());
      if (img.parts[s].stage.read(0, part[s].size(), part[s].data())) return -1;
    }
    std::vector<uint8_t> codes;
    std::vector<int64_t> ids;
    std::vector<int> head(S);
    auto id_of = [&](int s, int l, int j) {
      int64_t id;
      memcpy(&id, part[s].data() + at[s] + (size_t)img.parts[s].lens[l] * cb + (size_t)j * 8, 8);
      return ((id & ~kDelIdxMask) * S + s) | (id & kDelIdxMask);
    };
    for (int l = 0; ok && l < nlist; l++) {
      codes.resize((size_t)lens[l] * cb);
      ids.resize(lens[l]);
      std::fill(head.begin(), head.end(), 0);
      for (int j = 0; j < lens[l]; j++) {
        int best = -1;
        int64_t best_id = 0;
        for (int s = 0; s < S; s++) {
          if (head[s] >= img.parts[s].lens[l]) continue;
          const int64_t id = id_of(s, l, head[s]);
          if (best < 0 || (id & ~kDelIdxMask) < (best_id & ~kDelIdxMask)) best = s, best_id = id;
        }
        memcpy(codes.data() + (size_t)j * cb, part[best].data() + at[best] + (size_t)head[best] * cb, cb);
        ids[j] = best_id;
        head[best]++;
      }
      for (int s = 0; s < S; s++) at[s] += (size_t)img.parts[s].lens[l] * (cb + 8);
      ok = wr_bytes(f, codes.data(), codes.size()) && wr_bytes(f, ids.data(), ids.size() * 8);
    }
  }
  if (ok && img.indexed_count) ok = wr<int32_t>(f, (int32_t)img.indexed);  // ivfflat.cc:835
  if (!ok || fflush(f)) return fail("write error in " + path);
  return 0;
}

int IVFPQIndex::dump_gamma_extra(FILE* f) {
  std::vector<float> pq((size_t)M_ * ksub_ * dsub_);
  if (get_pq_centroids(pq.data())) return -1;
  // by_residual, code_size, write_product_quantizer (ivfpq.cc:1037-1039, index_io.cc:92-98)
  bool ok = wr<uint8_t>(f, 1) && wr<uint64_t>(f, (uint64_t)code_bytes()) && wr<uint64_t>(f, (uint64_t)d_) &&
            wr<uint64_t>(f, (uint64_t)M_) && wr<uint64_t>(f, (uint64_t)nbits_) && wr<uint64_t>(f, (uint64_t)pq.size()) &&
            wr_bytes(f, pq.data(), pq.size() * 4);
  if (ok && has_opq()) {  // write_opq (index_io.cc:230-246): "LTra", have_bias, A, b, d_in, d_out, is_trained
    std::vector<float> A((size_t)d_ * d_);
    if (get_opq(A.data())) return -1;
    ok = wr<uint32_t>(f, fourcc("LTra")) && wr<uint8_t>(f, 0) && wr<uint64_t>(f, (uint64_t)A.size()) &&
         wr_bytes(f, A.data(), A.size() * 4) && wr<uint64_t>(f, 0) && wr<int32_t>(f, d_) && wr<int32_t>(f, d_) &&
         wr<uint8_t>(f, 1);
  }
  return ok ? 0 : -1;
}

int IVFPQFastScanIndex::dump_gamma_extra(FILE* f) {
  std::vector<float> pq((size_t)M_ * ksub_ * dsub_);
  if (get_pq_centroids(pq.data())) return -1;
  const bool ok = wr<uint64_t>(f, (uint64_t)code_bytes()) && wr<uint64_t>(f, (uint64_t)d_) && wr<uint64_t>(f, (uint64_t)M_) &&
                  wr<uint64_t>(f, 4) && wr<uint64_t>(f, (uint64_t)pq.size()) && wr_bytes(f, pq.data(), pq.size() * 4);
  return ok ? 0 : -1;
}

int RaBitQIndex::dump_gamma_extra(FILE* f) {
  return wr<uint64_t>(f, (uint64_t)code_bytes()) && wr<int32_t>(f, nb_bits_) && wr<int32_t>(f, qb_) ? 0 : -1;
}

int VearchIndex::dump_gamma_extra(FILE* f) {
  std::vector<float> cb((size_t)16 * d_);
  if (get_codebook(cb.data())) return -1;
  const bool ok = wr<uint64_t>(f, (uint64_t)code_bytes()) && wr<int32_t>(f, mp_.nsubvector) && wr<int32_t>(f, nb_) &&
                  wr<double>(f, mp_.ns_threshold) && wr<uint8_t>(f, mp_.reordering ? 1 : 0) &&
                  wr<uint64_t>(f, (uint64_t)cb.size()) && wr_bytes(f, cb.data(), cb.size() * 4);
  return ok ? 0 : -1;
}

int BinaryIvfIndex::dump_gamma_extra(FILE* f) {
  std::vector<uint8_t> bc((size_t)nlist_ * cb_);
  if (get_binary_centroids(bc.data())) return -1;
  return wr<uint64_t>(f, (uint64_t)cb_) && wr<uint64_t>(f, (uint64_t)bc.size()) && wr_bytes(f, bc.data(), bc.size()) ? 0 : -1;
}

// ---- Load -----------------------------------------------------------------------------------
int IvfIndex::load_gamma(const std::string& dir, const std::string& abs_name, int64_t* load_num) {
  const bool was_trained = trained_;
  int64_t file_indexed = 0;
  const int rc = load_gamma_part(dir, abs_name, store_->size(), load_num, &file_indexed);
  // A refused file of a type whose trained state lives only in that file leaves no part of it behind: the index is
  // untrained again (its centroids may have been taken before the refusal), so it trains from the raw rows.
  if (rc && !was_trained && trained_ && !persists_trained_state()) {
    const std::string why = last_error();
    reset_index();
    set_last_error(why);
  }
  return rc;
}

int IvfIndex::load_gamma_part(const std::string& dir, const std::string& abs_name, int64_t store_rows, int64_t* load_num,
                              int64_t* file_indexed) {
  *load_num = 0;
  *file_indexed = 0;
  const GammaFileFormat gf = gamma_format();
  if (!gf.file) return 0;
  const std::string path = dir + "/" + abs_name + "/" + gf.file;
  FilePtr fp(fopen(path.c_str(), "rb"));
  FILE* f = fp.get();
  if (!f) return 0;  // "isn't existed, skip loading": it should train again after load (ivfflat.cc:846-850)
  std::lock_guard<std::mutex> bg(build_mu_);
  cudaSetDevice(device_);
  if (lists_ && lists_->total() > 0) return fail("load into a non-empty index");
  uint32_t h = 0;
  if (!rd(f, &h) || h != gf.magic) return fail("bad magic in " + path);
  IndexHeader ih, qh;
  uint64_t nlist = 0, nprobe = 0, n = 0;
  if (!rd_index_header(f, &ih) || !rd(f, &nlist) || !rd(f, &nprobe)) return fail("truncated ivf header in " + path);
  if (ih.d != d_ || (int64_t)nlist != nlist_)
    return fail("index file does not match the table: d=" + std::to_string(ih.d) + " nlist=" + std::to_string(nlist));
  if ((ih.metric == 1 ? kMetricL2 : kMetricIP) != mp_.metric) return fail("index file metric differs from the table's");
  if (!rd(f, &h)) return fail("truncated quantizer in " + path);
  if (h == fourcc("IHNf")) {
    // IndexHNSWFlat coarse quantizer (quantizer_type 1, gamma_index_ivfflat.cc:252-263): index header,
    // the HNSW graph (write_hnsw, index_io.cc:196-212: five vectors, five ints), then the IndexFlat that
    // stores the centroids.  The graph only approximates "nearest centroids"; this engine finds them
    // exactly with one dense tensor-core contraction, so the graph is skipped and the centroids are kept.
    IndexHeader hh;
    if (!rd_index_header(f, &hh)) return fail("truncated HNSW quantizer in " + path);
    const size_t elem[5] = {8, 4, 4, 8, 4};  // assign_probas, cum_nneighbor_per_level, levels, offsets, neighbors
    for (size_t e : elem) {
      uint64_t cnt = 0;
      if (!rd(f, &cnt) || cnt > ((uint64_t)1 << 40) || fseek(f, (long)(cnt * e), SEEK_CUR)) return fail("bad HNSW graph in " + path);
    }
    int32_t scalars[5];  // entry_point, max_level, efConstruction, efSearch, (deprecated) upper_beam
    if (!rd_bytes(f, scalars, sizeof scalars) || !rd(f, &h)) return fail("truncated HNSW quantizer in " + path);
  }
  if (h != fourcc("IxF2") && h != fourcc("IxFI") && h != fourcc("IxFl"))
    return fail("unsupported coarse quantizer in " + path + " (IndexFlat, or IndexHNSWFlat over IndexFlat)");
  if (!rd_index_header(f, &qh) || !rd(f, &n) || qh.d != d_ || qh.ntotal != nlist_ || n != (uint64_t)nlist_ * d_)
    return fail("bad quantizer in " + path);
  std::vector<float> cent((size_t)nlist_ * d_);
  if (!rd_bytes(f, cent.data(), cent.size() * 4)) return fail("truncated quantizer in " + path);
  uint8_t dm_type = 0;
  if (!rd(f, &dm_type) || !rd(f, &n)) return fail("truncated direct map in " + path);
  if (dm_type != 0 || n != 0) return fail("direct maps are not supported");  // gamma never maintains one
  if (set_centroids(cent.data(), nlist_)) return -1;
  if (load_gamma_extra(f)) return -1;
  if (spilled()) {
    double lambda = 0;
    if (!rd(f, &lambda)) return fail("truncated soar_lambda in " + path);
    if (lambda != mp_.soar_lambda)
      return fail("index file soar_lambda " + std::to_string(lambda) + " differs from the table's " +
                  std::to_string(mp_.soar_lambda));
  }
  // ReadInvertedLists (index_io.cc:143-194)
  uint32_t lt = 0;
  uint64_t nb = 0, cb = 0, ns = 0;
  if (!rd(f, &h) || !rd(f, &nb) || !rd(f, &cb) || !rd(f, &lt) || h != fourcc("ilar") || lt != fourcc("full"))
    return fail("bad inverted-list header in " + path);
  if (nb != (uint64_t)nlist_ || cb != gf.code_size) {
    // kIndexError: "unsupported inverted list format, it need rebuilding!" (ivfflat.cc:866-869)
    indexed_count_ = 0;
    return 0;
  }
  if (!rd(f, &ns) || ns != nb) return fail("bad inverted-list sizes in " + path);
  std::vector<uint64_t> sizes(nlist_);
  if (!rd_bytes(f, sizes.data(), sizes.size() * 8)) return fail("truncated inverted-list sizes in " + path);
  std::vector<int> add(nlist_);
  for (int l = 0; l < nlist_; l++) {
    if (sizes[l] > (uint64_t)INT32_MAX) return fail("inverted list too long");
    add[l] = (int)sizes[l];
  }
  // a shard keeps the entries whose global vid it owns: count them first, so its lists reserve no more than they take
  const int64_t S = shard_count_;
  auto mine = [&](int64_t id) { return (id & ~kDelIdxMask) % S == shard_id_; };
  std::vector<int64_t> ids;
  if (S > 1) {
    const long lists_at = ftell(f);
    for (int l = 0; l < nlist_; l++) {
      if (!sizes[l]) continue;
      ids.resize(sizes[l]);
      if (fseek(f, (long)(sizes[l] * cb), SEEK_CUR) || !rd_bytes(f, ids.data(), sizes[l] * 8))
        return fail("truncated list in " + path);
      add[l] = (int)std::count_if(ids.begin(), ids.end(), mine);
    }
    if (lists_at < 0 || fseek(f, lists_at, SEEK_SET)) return fail("cannot seek in " + path);
  }
  cudaStream_t st = build_stream_;
  {
    std::unique_lock<std::shared_mutex> lk(mu_);
    if (lists_->reserve(add, st)) return -1;
  }
  std::vector<uint8_t> codes, padded;
  int64_t live = 0, max_vid = -1;
  VidSlots v2p(copies());  // installed only if the whole file loads
  std::vector<int> dead(nlist_, 0);
  const size_t my_cb = (size_t)code_bytes();
  for (int l = 0; l < nlist_; l++) {
    size_t len = sizes[l];
    if (!len) continue;
    codes.resize(len * cb);
    ids.resize(len);
    if (!rd_bytes(f, codes.data(), codes.size()) || !rd_bytes(f, ids.data(), len * 8)) return fail("truncated list in " + path);
    if (S > 1) {  // this shard's entries in file order, as local vids, tombstone bits kept
      size_t w = 0;
      for (size_t r = 0; r < len; r++) {
        if (!mine(ids[r])) continue;
        if (w != r) memmove(codes.data() + w * cb, codes.data() + r * cb, cb);
        ids[w++] = ((ids[r] & ~kDelIdxMask) / S) | (ids[r] & kDelIdxMask);
      }
      len = w;
      if (!len) continue;
    }
    const uint8_t* src = codes.data();
    if (my_cb != cb) {  // padded rows in memory
      padded.assign(len * my_cb, 0);
      for (size_t r = 0; r < len; r++) memcpy(padded.data() + r * my_cb, codes.data() + r * cb, cb);
      src = padded.data();
    }
    GB_CUDA(cudaMemcpyAsync(lists_->list_data(l), src, len * my_cb, cudaMemcpyHostToDevice, st));
    GB_CUDA(cudaMemcpyAsync(lists_->list_ids(l), ids.data(), len * 8, cudaMemcpyHostToDevice, st));
    GB_CUDA(cudaStreamSynchronize(st));  // the staging vectors are reused by the next list
    for (size_t pos = 0; pos < len; pos++) {
      const int64_t id = ids[pos];
      if (id < 0) {  // deleted_nums_[bno]++ (index_io.cc:178-181)
        dead[l]++;
        continue;
      }
      live++;
      max_vid = std::max(max_vid, id);
      if (id >= v2p.size()) v2p.grow(std::max(id + 1, v2p.size() * 2));
      // the vid's live entries in file order fill its slots; an unspilled vid's later entry replaces the earlier one
      uint64_t* at = v2p.at(id);
      int c = 0;
      while (c + 1 < copies() && at[c] != VidSlots::kNone) c++;
      if (c > 0 && at[c] != VidSlots::kNone) return fail("vid " + std::to_string(id) + " has more than two live entries in " + path);
      for (int j = 0; j < c; j++)
        if ((at[j] >> 32) == (uint64_t)l) return fail("vid " + std::to_string(id) + " has two live entries in list " + std::to_string(l) + " of " + path);
      at[c] = (uint64_t)l << 32 | (uint64_t)pos;
    }
  }
  int64_t indexed = live;  // IwPQ: ReadInvertedLists' running count (total - tombstones)
  *file_indexed = live;
  if (gf.indexed_count) {
    int32_t cnt = 0;
    if (!rd(f, &cnt) || cnt < 0) return fail("invalid indexed count in " + path);  // ivfflat.cc:871-878
    *file_indexed = cnt;
    indexed = cnt > shard_id_ ? (cnt - shard_id_ + S - 1) / S : 0;  // the vids below cnt this shard owns
  }
  const int64_t rows = store_rows > shard_id_ ? (store_rows - shard_id_ + S - 1) / S : 0;
  if (indexed > rows || max_vid >= rows || *file_indexed > store_rows)
    return fail("index file covers " + std::to_string(std::max(*file_indexed, global_vid(max_vid) + 1)) +
                " vectors, the vector store holds " + std::to_string(store_rows));
  {  // publish: nothing above this point changed what a search can see
    std::unique_lock<std::shared_mutex> lk(mu_);
    if (lists_->commit(add, st)) return -1;
    std::swap(slots_, v2p);
    for (int l = 0; l < nlist_; l++) lists_->add_dead(l, dead[l]);
    if (lists_changed(st)) return -1;  // IVF-Flat on a host store: the row pointers into the loaded lists
    GB_CUDA(cudaStreamSynchronize(st));
  }
  indexed_count_ = indexed;
  *load_num = indexed;
  return 0;
}

int IVFPQIndex::load_gamma_extra(FILE* f) {
  uint8_t by_residual = 0;
  uint64_t code_size = 0, d = 0, M = 0, nbits = 0, n = 0;
  if (!rd(f, &by_residual) || !rd(f, &code_size) || !rd(f, &d) || !rd(f, &M) || !rd(f, &nbits) || !rd(f, &n))
    return fail("truncated product quantizer");
  if (!by_residual) return fail("by_residual = false is not supported");
  if (d != (uint64_t)d_ || M != (uint64_t)M_ || nbits != (uint64_t)nbits_ || code_size != (uint64_t)code_bytes() ||
      n != (uint64_t)M_ * ksub_ * dsub_)
    return fail("product quantizer does not match the table: d=" + std::to_string(d) + " M=" + std::to_string(M) +
                " nbits=" + std::to_string(nbits) + " code_size=" + std::to_string(code_size) + " centroids=" +
                std::to_string(n) + " (table: d=" + std::to_string(d_) + " M=" + std::to_string(M_) + " nbits=" +
                std::to_string(nbits_) + " code_size=" + std::to_string(code_bytes()) + ")");
  std::vector<float> pq((size_t)n);
  if (!rd_bytes(f, pq.data(), pq.size() * 4)) return fail("truncated product quantizer");
  if (has_opq()) {  // read_opq (index_io.cc:248-270); whether the block is there is decided by the table's params
    uint32_t h = 0;
    uint8_t have_bias = 0, trained = 0;
    uint64_t na = 0, nb = 0;
    int32_t din = 0, dout = 0;
    if (!rd(f, &h) || h != fourcc("LTra") || !rd(f, &have_bias) || !rd(f, &na) || na != (uint64_t)d_ * d_)
      return fail("bad OPQ block (table has opq, file does not match)");
    std::vector<float> A((size_t)na);
    if (!rd_bytes(f, A.data(), A.size() * 4) || !rd(f, &nb) || fseek(f, (long)(nb * 4), SEEK_CUR) || !rd(f, &din) ||
        !rd(f, &dout) || !rd(f, &trained) || din != d_ || dout != d_ || have_bias)
      return fail("bad OPQ block");
    if (set_opq(A.data())) return -1;
  }
  return set_pq_centroids(pq.data());  // also recomputes the precomputed table (ivfpq.cc:1093-1095)
}

int IVFPQFastScanIndex::load_gamma_extra(FILE* f) {
  uint64_t code_size = 0, d = 0, M = 0, nbits = 0, n = 0;
  if (!rd(f, &code_size) || !rd(f, &d) || !rd(f, &M) || !rd(f, &nbits) || !rd(f, &n)) return fail("truncated IVFPQFastScan codebook");
  if (d != (uint64_t)d_ || M != (uint64_t)M_ || nbits != 4 || code_size != (uint64_t)code_bytes() ||
      n != (uint64_t)M_ * ksub_ * dsub_)
    return fail("IVFPQFastScan codebook does not match the table: d=" + std::to_string(d) + " M=" + std::to_string(M) +
                " nbits=" + std::to_string(nbits) + " code_size=" + std::to_string(code_size) + " (table: d=" +
                std::to_string(d_) + " M=" + std::to_string(M_) + " nbits=4)");
  std::vector<float> pq((size_t)n);
  if (!rd_bytes(f, pq.data(), pq.size() * 4)) return fail("truncated IVFPQFastScan codebook");
  return set_pq_centroids(pq.data());
}

int RaBitQIndex::load_gamma_extra(FILE* f) {
  uint64_t code_size = 0;
  int32_t nb_bits = 0, qb = 0;
  if (!rd(f, &code_size) || !rd(f, &nb_bits) || !rd(f, &qb)) return fail("truncated IVFRABITQ parameters");
  if (nb_bits != nb_bits_ || qb != qb_ || code_size != (uint64_t)code_bytes())
    return fail("IVFRABITQ parameters do not match the table: nb_bits=" + std::to_string(nb_bits) + " qb=" +
                std::to_string(qb) + " code_size=" + std::to_string(code_size) + " (table: nb_bits=" +
                std::to_string(nb_bits_) + " qb=" + std::to_string(qb_) + ")");
  return 0;  // the codes depend on the centroids and nb_bits alone: no rotation, no seed
}

int VearchIndex::load_gamma_extra(FILE* f) {
  uint64_t code_size = 0, n = 0;
  int32_t nsub = 0, nb = 0;
  double t = 0;
  uint8_t reordering = 0;
  if (!rd(f, &code_size) || !rd(f, &nsub) || !rd(f, &nb) || !rd(f, &t) || !rd(f, &reordering) || !rd(f, &n))
    return fail("truncated VEARCH codebook");
  const bool same_t = (isnan(t) && isnan(mp_.ns_threshold)) || t == mp_.ns_threshold;
  if (nsub != mp_.nsubvector || nb != nb_ || !same_t || (reordering != 0) != mp_.reordering ||
      code_size != (uint64_t)code_bytes() || n != (uint64_t)16 * d_)
    return fail("VEARCH codebook does not match the table: nsubvector=" + std::to_string(nsub) + " blocks=" +
                std::to_string(nb) + " ns_threshold=" + std::to_string(t) + " reordering=" + std::to_string(reordering) +
                " (table: nsubvector=" + std::to_string(mp_.nsubvector) + " blocks=" + std::to_string(nb_) +
                " ns_threshold=" + std::to_string(mp_.ns_threshold) + " reordering=" + std::to_string(mp_.reordering) + ")");
  std::vector<float> cb((size_t)n);
  if (!rd_bytes(f, cb.data(), cb.size() * 4)) return fail("truncated VEARCH codebook");
  return set_codebook(cb.data());
}

int BinaryIvfIndex::load_gamma_extra(FILE* f) {
  uint64_t code_size = 0, n = 0;
  if (!rd(f, &code_size) || !rd(f, &n)) return fail("truncated BINARYIVF centroids");
  if (code_size != (uint64_t)cb_ || n != (uint64_t)nlist_ * cb_)
    return fail("BINARYIVF centroids do not match the table: code_size=" + std::to_string(code_size) +
                " (table: " + std::to_string(cb_) + ")");
  std::vector<uint8_t> bc((size_t)n);
  if (!rd_bytes(f, bc.data(), bc.size())) return fail("truncated BINARYIVF centroids");
  // the packed centroids as they were, not re-derived from the float ones (set_binary_centroids may have set them alone)
  return set_binary_centroids(bc.data(), nlist_);
}

}  // namespace gb
