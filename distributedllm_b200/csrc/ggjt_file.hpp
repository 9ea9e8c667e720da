// ggjt_file.hpp -- read-only view of a reference slice / extra-layers file (GGJT v3 + first_layer).
// Byte layout: distllm/slice_model.cpp:239-302 (writer), distllm/tensor_processor.cpp:152-248 (reader).
#pragma once
#include <cstdint>
#include <cstring>
#include <map>
#include <stdexcept>
#include <string>
#include <vector>
#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

namespace b200 {

enum GgmlType : uint32_t { GT_F32 = 0, GT_F16 = 1, GT_Q4_0 = 2, GT_Q4_1 = 3, GT_Q5_0 = 6, GT_Q5_1 = 7, GT_Q8_0 = 8,
                         GT_Q2_K = 10, GT_Q3_K = 11, GT_Q4_K = 12, GT_Q5_K = 13, GT_Q6_K = 14 };

struct GgjtTensor {
    std::string name;
    uint32_t type = 0;
    std::vector<uint32_t> ne;       // ne[0] = row length
    size_t offset = 0, nbytes = 0;
};

struct GgjtFile {
    int fd = -1;
    const uint8_t * base = nullptr;
    size_t size = 0;
    uint32_t n_vocab = 0, n_embd = 0, n_mult = 0, n_head = 0, n_layer = 0, n_rot = 0, first_layer = 0, ftype = 0;
    std::vector<std::pair<std::string, float>> vocab;
    std::vector<GgjtTensor> tensors;
    std::map<std::string, size_t> index;

    static size_t type_bytes(uint32_t type, size_t nelem) {
        switch (type) {
            case GT_F32:  return nelem * 4;
            case GT_F16:  return nelem * 2;
            case GT_Q4_0: return nelem / 32 * 18;
            case GT_Q4_1: return nelem / 32 * 20;
            case GT_Q5_0: return nelem / 32 * 22;
            case GT_Q5_1: return nelem / 32 * 24;
            case GT_Q8_0: return nelem / 32 * 34;
            case GT_Q2_K: return nelem / 256 * 84;
            case GT_Q3_K: return nelem / 256 * 110;
            case GT_Q4_K: return nelem / 256 * 144;
            case GT_Q5_K: return nelem / 256 * 176;
            case GT_Q6_K: return nelem / 256 * 210;
            default: throw std::runtime_error("unrecognized tensor type " + std::to_string(type));
        }
    }

    // A throwing constructor never runs the destructor: parse() may throw on a malformed file, so the fd and the
    // mapping are released here before the exception leaves (a long-running node must not leak them per bad upload).
    explicit GgjtFile(const std::string & path, bool keep_vocab) {
        try { parse(path, keep_vocab); }
        catch (...) { release(); throw; }
    }
    void release() {
        if (base) { munmap((void *) base, size); base = nullptr; }
        if (fd >= 0) { ::close(fd); fd = -1; }
    }
    void parse(const std::string & path, bool keep_vocab) {
        fd = ::open(path.c_str(), O_RDONLY);
        if (fd < 0) throw std::runtime_error("cannot open " + path);
        struct stat st;
        if (fstat(fd, &st) != 0 || st.st_size <= 0) throw std::runtime_error("cannot stat (or empty file) " + path);
        size = (size_t) st.st_size;
        void * p = mmap(nullptr, size, PROT_READ, MAP_PRIVATE, fd, 0);
        if (p == MAP_FAILED) throw std::runtime_error("mmap failed for " + path);
        base = (const uint8_t *) p;
        size_t pos = 0;
        auto u32 = [&]() -> uint32_t {
            if (pos + 4 > size) throw std::runtime_error("unexpected end of file in " + path);
            uint32_t v; memcpy(&v, base + pos, 4); pos += 4; return v;
        };
        const uint32_t magic = u32();
        const uint32_t version = u32();
        if (magic != 0x67676a74u || version != 3)
            throw std::runtime_error("unknown (magic, version) combination; expected a GGJT v3 slice file: " + path);
        n_vocab = u32(); n_embd = u32(); n_mult = u32(); n_head = u32(); n_layer = u32(); n_rot = u32();
        first_layer = u32(); ftype = u32();
        if (keep_vocab) vocab.reserve(n_vocab);
        for (uint32_t i = 0; i < n_vocab; i++) {
            const uint32_t len = u32();
            if (pos + len + 4 > size) throw std::runtime_error("truncated vocabulary in " + path);
            if (keep_vocab) {
                float score; memcpy(&score, base + pos + len, 4);
                vocab.emplace_back(std::string((const char *) base + pos, len), score);
            }
            pos += len + 4;
        }
        while (pos < size) {
            GgjtTensor t;
            const uint32_t n_dims = u32(), name_len = u32();
            t.type = u32();
            if (n_dims < 1 || n_dims > 2) throw std::runtime_error("tensor should not be " + std::to_string(n_dims) + "-dimensional");
            size_t nelem = 1;
            for (uint32_t d = 0; d < n_dims; d++) { t.ne.push_back(u32()); nelem *= t.ne.back(); }
            if (pos + name_len > size) throw std::runtime_error("truncated tensor record in " + path);
            t.name.assign((const char *) base + pos, name_len); pos += name_len;
            pos = (pos + 31) & ~(size_t) 31;
            t.offset = pos; t.nbytes = type_bytes(t.type, nelem);
            if (pos + t.nbytes > size) throw std::runtime_error("tensor '" + t.name + "' runs past the end of " + path);
            pos += t.nbytes;
            index[t.name] = tensors.size();
            tensors.push_back(std::move(t));
        }
    }
    ~GgjtFile() { release(); }
    GgjtFile(const GgjtFile &) = delete;
    GgjtFile & operator=(const GgjtFile &) = delete;

    // tensor by name with the shape check of llama_model_loader::get_tensor (tensor_processor.cpp:950-963)
    const GgjtTensor & get(const std::string & name, const std::vector<uint32_t> & ne) const {
        auto it = index.find(name);
        if (it == index.end()) throw std::runtime_error("tensor '" + name + "' is missing from model");
        const GgjtTensor & t = tensors[it->second];
        if (t.ne != ne) throw std::runtime_error("tensor '" + name + "' has wrong shape");
        return t;
    }
    const uint8_t * data(const GgjtTensor & t) const { return base + t.offset; }
};

// Read-only view of a LoRA adapter file (`ggla` v1), as convert-lora-to-ggml.py:49-74,111-131 writes it and
// llama_apply_lora_from_file_internal (llama.cpp:2846-2960) reads it: magic, version, r, alpha (i32), then per tensor
// n_dims, name_len, ftype (0 F32, 1 F16), ne[n_dims], the name, and the data at the next multiple of 32 bytes.
// Only the layout is checked here; what the tensors may be is the loader's business.
struct GglaFile {
    int fd = -1;
    const uint8_t * base = nullptr;
    size_t size = 0;
    int32_t r = 0, alpha = 0;
    std::vector<GgjtTensor> tensors;    // file order; ne holds n_dims entries

    explicit GglaFile(const std::string & path) {
        try { parse(path); }
        catch (...) { release(); throw; }
    }
    void release() {
        if (base) { munmap((void *) base, size); base = nullptr; }
        if (fd >= 0) { ::close(fd); fd = -1; }
    }
    void parse(const std::string & path) {
        fd = ::open(path.c_str(), O_RDONLY);
        if (fd < 0) throw std::runtime_error("cannot open adapter " + path);
        struct stat st;
        if (fstat(fd, &st) != 0 || st.st_size <= 0) throw std::runtime_error("cannot stat (or empty file) adapter " + path);
        size = (size_t) st.st_size;
        void * p = mmap(nullptr, size, PROT_READ, MAP_PRIVATE, fd, 0);
        if (p == MAP_FAILED) throw std::runtime_error("mmap failed for adapter " + path);
        base = (const uint8_t *) p;
        size_t pos = 0;
        auto u32 = [&](const char * what) -> uint32_t {
            if (pos + 4 > size) throw std::runtime_error(std::string("adapter truncated in ") + what + ": " + path);
            uint32_t v; memcpy(&v, base + pos, 4); pos += 4; return v;
        };
        const uint32_t magic = u32("the header"), version = u32("the header");
        if (magic != 0x67676c61u) throw std::runtime_error("bad magic: not a ggla adapter file: " + path);
        if (version != 1) throw std::runtime_error("unsupported ggla version " + std::to_string(version) + " (expected 1): " + path);
        r = (int32_t) u32("the header"); alpha = (int32_t) u32("the header");
        if (r <= 0) throw std::runtime_error("adapter rank r = " + std::to_string(r) + " is not positive: " + path);
        while (pos < size) {
            GgjtTensor t;
            const uint32_t n_dims = u32("a tensor record"), name_len = u32("a tensor record");
            t.type = u32("a tensor record");
            if (n_dims < 1 || n_dims > 4 || name_len > 1024)
                throw std::runtime_error("malformed tensor record at byte " + std::to_string(pos - 12) + " (n_dims " +
                                         std::to_string(n_dims) + ", name length " + std::to_string(name_len) + ")");
            size_t nelem = 1;
            for (uint32_t d = 0; d < n_dims; d++) { t.ne.push_back(u32("a tensor record")); nelem *= t.ne.back(); }
            if (pos + name_len > size) throw std::runtime_error("adapter truncated in a tensor name: " + path);
            t.name.assign((const char *) base + pos, name_len); pos += name_len;
            if (t.type != GT_F32 && t.type != GT_F16)
                throw std::runtime_error("tensor '" + t.name + "' has ftype " + std::to_string(t.type) + " (0 = F32, 1 = F16)");
            pos = (pos + 31) & ~(size_t) 31;
            t.offset = pos; t.nbytes = nelem * (t.type == GT_F32 ? 4 : 2);
            if (pos + t.nbytes > size) throw std::runtime_error("tensor '" + t.name + "' runs past the end of " + path);
            pos += t.nbytes;
            tensors.push_back(std::move(t));
        }
    }
    ~GglaFile() { release(); }
    GglaFile(const GglaFile &) = delete;
    GglaFile & operator=(const GglaFile &) = delete;
    const uint8_t * data(const GgjtTensor & t) const { return base + t.offset; }
};

}  // namespace b200
