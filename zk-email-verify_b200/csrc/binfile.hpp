// iden3 binfile container (`.zkey`, `.ptau`, `.wtns`, `.r1cs`): magic[4], u32 version, u32 nSections, then
// {u32 type, u64 size, payload} per section, everything little-endian.  Host only.
#pragma once
#include <cstdint>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

namespace zke {

struct SecView { const uint8_t* p = nullptr; size_t n = 0; };
struct BinSection { uint32_t type; SecView view; };

inline uint32_t rd32(const uint8_t* p) { uint32_t v; memcpy(&v, p, 4); return v; }
inline uint64_t rd64(const uint8_t* p) { uint64_t v; memcpy(&v, p, 8); return v; }

// The sections of a container of len >= 12 bytes, in file order.  The caller checks the magic and the version first,
// and the section types and contents after; `file` (".zkey", ...) names the format in the truncation errors.
inline std::vector<BinSection> binfile_sections(const uint8_t* b, size_t len, const char* file) {
    std::vector<BinSection> out;
    const uint32_t n_sec = rd32(b + 8);
    size_t pos = 12;
    for (uint32_t i = 0; i < n_sec; ++i) {
        if (len - pos < 12) throw std::runtime_error(std::string("truncated ") + file + " (section header)");
        const uint32_t type = rd32(b + pos);
        const uint64_t size = rd64(b + pos + 4);
        pos += 12;
        if (size > len - pos) throw std::runtime_error(std::string("truncated ") + file + " (section " + std::to_string(type) + ")");
        out.push_back(BinSection{type, SecView{b + pos, (size_t)size}});
        pos += (size_t)size;
    }
    return out;
}

// appends iden3 binfile pieces to a caller buffer
struct BinWriter {
    uint8_t* p;
    void u32(uint32_t v) { memcpy(p, &v, 4); p += 4; }
    void u64(uint64_t v) { memcpy(p, &v, 8); p += 8; }
    void bytes(const void* src, size_t n) { memcpy(p, src, n); p += n; }
    void header(const char* magic, uint32_t version, uint32_t n_sections) { bytes(magic, 4); u32(version); u32(n_sections); }
    void section(int s, size_t size) { u32((uint32_t)s); u64(size); }
};

}  // namespace zke
