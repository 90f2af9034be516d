// p3gpu.hpp — header-only C++ host mirror of the reference's trait surfaces over the C ABI in p3gpu.h.
//
// The reference's host code is Rust; this is the C++ equivalent of the shim in
// INTEGRATION.md: same names, argument meaning and error behaviour (prover-side shape errors throw, where the
// reference panics).  Matrices are caller-owned row-major uint32_t buffers in Montgomery form.
//   p3gpu::Radix2DitParallel  ~ TwoAdicSubgroupDft          dft/src/traits.rs:28-291, radix_2_dit_parallel.rs:144-246
//   p3gpu::MerkleTreeMmcs     ~ Mmcs::commit                merkle-tree/src/mmcs/batch.rs:42-64
//   p3gpu::TwoAdicFriFolding  ~ FriFoldingStrategy          fri/src/two_adic_pcs.rs:134-213
//   p3gpu::TwoAdicFriPcs      ~ Pcs::commit (host trace in, LDE + tree resident on the device)   fri/src/two_adic_pcs.rs:300-324
//   p3gpu::MerkleTreeMmcs::open_multi_batch / prune_paths ~ Mmcs::open_multi_batch     merkle-tree/src/mmcs/mod.rs:276-428, pruning.rs
#pragma once
#include <algorithm>
#include <cstdint>
#include <map>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "p3gpu.h"

namespace p3gpu {

struct Error : std::runtime_error { using std::runtime_error::runtime_error; };
inline void check(int32_t rc) {
    if (rc != P3GPU_OK) throw Error("p3gpu error " + std::to_string(rc) + ": " + p3gpu_last_error());
}

class Context {
  public:
    explicit Context(int device = 0) { check(p3gpu_ctx_create(device, &ctx_)); }
    ~Context() { p3gpu_ctx_destroy(ctx_); }
    Context(const Context &) = delete;
    Context &operator=(const Context &) = delete;
    p3gpu_ctx *raw() const { return ctx_; }
  private:
    p3gpu_ctx *ctx_ = nullptr;
};

// Device memory owned by the host object that holds it (p3gpu_malloc / p3gpu_free)
class DeviceBuffer {
  public:
    DeviceBuffer() = default;
    DeviceBuffer(Context &c, size_t words) : c_(&c), words_(words) { void *p = nullptr; check(p3gpu_malloc(c.raw(), std::max<size_t>(words, 1) * 4, &p)); ptr_ = (uint32_t *)p; }
    ~DeviceBuffer() { if (ptr_) p3gpu_free(c_->raw(), ptr_); }
    DeviceBuffer(DeviceBuffer &&o) noexcept : c_(o.c_), ptr_(o.ptr_), words_(o.words_) { o.ptr_ = nullptr; }
    DeviceBuffer &operator=(DeviceBuffer &&o) noexcept { std::swap(c_, o.c_); std::swap(ptr_, o.ptr_); std::swap(words_, o.words_); return *this; }
    DeviceBuffer(const DeviceBuffer &) = delete;
    DeviceBuffer &operator=(const DeviceBuffer &) = delete;
    uint32_t *data() const { return ptr_; }
    size_t words() const { return words_; }
    std::vector<uint32_t> to_host(size_t offset_words, size_t n_words) const {
        if (offset_words + n_words > words_) throw Error("device read out of bounds");
        std::vector<uint32_t> out(n_words);
        if (n_words) check(p3gpu_memcpy_d2h(c_->raw(), out.data(), ptr_ + offset_words, n_words * 4));
        return out;
    }
  private:
    Context *c_ = nullptr;
    uint32_t *ptr_ = nullptr;
    size_t words_ = 0;
};

struct RowMajorMatrix {                 // matrix/src/dense.rs:23-36
    std::vector<uint32_t> values;
    size_t width = 0;
    size_t height() const { return width ? values.size() / width : 0; }
};

// Result of the batch transforms: inner matrix holds the rows in bit-reversed order (matrix/src/bitrev.rs:82-101)
struct BitReversedMatrixView {
    RowMajorMatrix inner;
    RowMajorMatrix bit_reverse_rows() && { return std::move(inner); }   // zero data movement, as in the reference
};

class Radix2DitParallel {
  public:
    Radix2DitParallel(Context &c, int field) : c_(c), field_(field) {}
    RowMajorMatrix dft_batch(RowMajorMatrix m) const { return run(std::move(m), P3GPU_DFT, 0); }
    RowMajorMatrix idft_batch(RowMajorMatrix m) const { return run(std::move(m), P3GPU_IDFT, 0); }
    RowMajorMatrix coset_dft_batch(RowMajorMatrix m, uint32_t shift) const { return run(std::move(m), P3GPU_COSET_DFT, shift); }
    RowMajorMatrix coset_idft_batch(RowMajorMatrix m, uint32_t shift) const { return run(std::move(m), P3GPU_COSET_IDFT, shift); }
    BitReversedMatrixView coset_lde_batch(const RowMajorMatrix &m, unsigned added_bits, uint32_t shift) const {
        BitReversedMatrixView out;
        out.inner.width = m.width;
        out.inner.values.resize(m.values.size() << added_bits);
        check(p3gpu_coset_lde_batch(c_.raw(), field_, m.values.data(), m.height(), m.width, added_bits, shift,
                                    out.inner.values.data(), /*bitrev_rows=*/1));
        return out;
    }
  private:
    RowMajorMatrix run(RowMajorMatrix m, int kind, uint32_t shift) const {
        check(p3gpu_dft_batch(c_.raw(), field_, kind, m.values.data(), m.height(), m.width, shift));
        return m;
    }
    Context &c_;
    int field_;
};

struct MerkleTree {                     // merkle-tree/src/merkle_tree.rs:33-69 (arity schedule is all 2)
    std::vector<std::vector<uint32_t>> digest_layers;   // layer k: len_k * 8 words
    std::vector<uint32_t> cap(size_t cap_height) const {
        if (cap_height >= digest_layers.size()) throw Error("cap_height exceeds tree depth");
        const auto &l = digest_layers[digest_layers.size() - 1 - cap_height];
        size_t n = std::min<size_t>((size_t)1 << cap_height, l.size() / 8);
        return std::vector<uint32_t>(l.begin(), l.begin() + n * 8);
    }
};

// `hash`: one of the P3GPU_HASH_* kinds.  Every kind's digest is 8 words; for P3GPU_HASH_SHA256 and P3GPU_HASH_SHA256_COMPRESS
// they hold a [u8; 32] digest, the words' little-endian bytes being the digest's bytes in order.
class MerkleTreeMmcs {
  public:
    MerkleTreeMmcs(Context &c, int field, int hash, size_t cap_height) : c_(c), field_(field), hash_(hash), cap_height_(cap_height) {}
    // Mmcs::commit: returns (cap, tree)
    std::pair<std::vector<uint32_t>, MerkleTree> commit(const std::vector<const RowMajorMatrix *> &inputs) const {
        if (inputs.empty()) throw Error("No matrices given?");
        std::vector<const uint32_t *> ptrs; std::vector<size_t> hs, ws; size_t max_h = 0;
        for (auto *m : inputs) { ptrs.push_back(m->values.data()); hs.push_back(m->height()); ws.push_back(m->width); max_h = std::max(max_h, m->height()); }
        std::vector<uint32_t> flat(p3gpu_merkle_total_digests(max_h) * 8);
        size_t lens[65], n = 0;
        check(p3gpu_merkle_commit(c_.raw(), field_, hash_, ptrs.size(), ptrs.data(), hs.data(), ws.data(), flat.data(), lens, &n));
        MerkleTree t; size_t off = 0;
        for (size_t k = 0; k < n; k++) { t.digest_layers.emplace_back(flat.begin() + off * 8, flat.begin() + (off + lens[k]) * 8); off += lens[k]; }
        return {t.cap(std::min(cap_height_, n - 1)), std::move(t)};
    }
  private:
    Context &c_; int field_, hash_; size_t cap_height_;
};

// What Pcs::commit keeps for the rest of the proof: the committed LDE (bit-reversed rows) and every digest layer, on the device.
struct DeviceProverData {
    DeviceBuffer lde, layers;
    std::vector<size_t> layer_lens;     // digests per layer, layer 0 = leaves
    size_t height = 0, width = 0;       // of the LDE
};

// A multi-opening in the reference's wire shape (fri/src/proof.rs:68-75): opened_values[query] = the row, one pruned proof.
struct MultiOpening {
    std::vector<std::vector<uint32_t>> opened_values;
    std::vector<uint32_t> pruned_digests;   // k * 8 words, wire order of merkle-tree/src/pruning.rs:187-232
};

// prune_paths for the binary schedule: `paths` = n * levels * 8 words (sibling digests bottom-up per query).  The sorted distinct
// leaves fold up level by level; a node whose sibling is not on the frontier takes it from the smallest queried leaf below it.
inline std::vector<uint32_t> prune_paths(const std::vector<uint32_t> &indices, const std::vector<uint32_t> &paths, size_t levels) {
    if (paths.size() != indices.size() * levels * 8) throw Error("paths do not match indices x levels");
    std::map<uint32_t, size_t> first;
    for (size_t q = 0; q < indices.size(); q++) first.emplace(indices[q], q);
    std::vector<std::pair<uint64_t, size_t>> nodes(first.begin(), first.end()), parents;
    std::vector<uint32_t> out;
    for (size_t level = 0; level < levels; level++) {
        parents.clear();
        for (size_t k = 0; k < nodes.size();) {
            const uint64_t idx = nodes[k].first;
            const size_t lead = nodes[k].second;
            if (k + 1 < nodes.size() && nodes[k + 1].first == (idx ^ 1)) k += 2;
            else {
                const uint32_t *d = &paths[(lead * levels + level) * 8];
                out.insert(out.end(), d, d + 8);
                k += 1;
            }
            parents.emplace_back(idx >> 1, lead);
        }
        nodes.swap(parents);
    }
    return out;
}

class TwoAdicFriPcs {
  public:
    TwoAdicFriPcs(Context &c, int field, int hash, unsigned log_blowup, size_t cap_height)
        : c_(c), field_(field), hash_(hash), log_blowup_(log_blowup), cap_height_(cap_height) {}
    // Pcs::commit for one trace over the subgroup H: (cap, prover data).  The trace crosses PCIe once; only the cap comes back.
    std::pair<std::vector<uint32_t>, DeviceProverData> commit(const RowMajorMatrix &evals) const {
        const size_t h = evals.height(), w = evals.width, H = h << log_blowup_;
        if (h == 0 || (h & (h - 1))) throw Error("trace height must be a power of two");
        DeviceProverData pd;
        pd.height = H; pd.width = w;
        pd.lde = DeviceBuffer(c_, H * w);
        pd.layers = DeviceBuffer(c_, p3gpu_merkle_total_digests(H) * 8);
        size_t lens[65], n = 0, cap_len = 0;
        std::vector<uint32_t> cap(((size_t)1 << cap_height_) * 8);
        check(p3gpu_pcs_commit(c_.raw(), field_, hash_, evals.values.data(), h, w, log_blowup_, (unsigned)cap_height_, pd.lde.data(),
                               pd.layers.data(), lens, &n, cap.data(), &cap_len));
        pd.layer_lens.assign(lens, lens + n);
        cap.resize(cap_len * 8);
        return {std::move(cap), std::move(pd)};
    }
    // Mmcs::open_multi_batch on the committed data: rows gathered and paths walked on the device, pruned on the host
    MultiOpening open_multi_batch(const std::vector<uint32_t> &indices, const DeviceProverData &pd) const {
        const size_t n = indices.size(), nl = pd.layer_lens.size();
        for (uint32_t i : indices) if (i >= pd.height) throw Error("index out of bounds for height " + std::to_string(pd.height));
        const size_t eff = std::min(cap_height_, nl ? nl - 1 : 0), path_len = nl - 1 - eff;
        DeviceBuffer rows(c_, n * pd.width), paths(c_, n * path_len * 8);
        MultiOpening out;
        if (n == 0) return out;
        check(p3gpu_gather_rows_dev(c_.raw(), pd.lde.data(), pd.height, pd.width, indices.data(), n, 0, rows.data()));
        const std::vector<uint32_t> flat = rows.to_host(0, n * pd.width);
        for (size_t q = 0; q < n; q++) out.opened_values.emplace_back(flat.begin() + q * pd.width, flat.begin() + (q + 1) * pd.width);
        std::vector<uint32_t> full;
        if (path_len) {
            check(p3gpu_merkle_paths_dev(c_.raw(), pd.layers.data(), pd.layer_lens.data(), nl, path_len, indices.data(), n, 0, paths.data()));
            full = paths.to_host(0, n * path_len * 8);
        }
        out.pruned_digests = prune_paths(indices, full, path_len);
        return out;
    }
  private:
    Context &c_; int field_, hash_; unsigned log_blowup_; size_t cap_height_;
};

class TwoAdicFriFolding {
  public:
    TwoAdicFriFolding(Context &c, int field) : c_(c), field_(field) {}
    // fold_matrix: m = rows x (arity * 4) words (EF4 values, bit-reversed evaluation order) -> rows x 4 words
    std::vector<uint32_t> fold_matrix(const uint32_t beta[4], unsigned log_arity, const std::vector<uint32_t> &m) const {
        const size_t rows = (m.size() / 4) >> log_arity;
        std::vector<uint32_t> out(rows * 4);
        check(p3gpu_fri_fold(c_.raw(), field_, m.data(), rows, log_arity, beta, out.data()));
        return out;
    }
  private:
    Context &c_; int field_;
};

}  // namespace p3gpu
