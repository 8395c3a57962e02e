// bb_crc32.cuh — CRC-32 (gzip's polynomial, reflected) arithmetic shared by the BGZF compressor and inflater: threads
// compute the CRC register of their own slice of a member, and the registers are combined by moving each one past the
// bytes after its slice (multiplication by x^(8 n) modulo the polynomial).
#pragma once
#include <cstdint>

#define BGZF_POLY 0xedb88320u

// a * b modulo the CRC-32 polynomial, both reflected (bit 31 is x^0)
__device__ __forceinline__ uint32_t bgzf_mulmod(uint32_t a, uint32_t b) {
    uint32_t p = 0;
    for (int i = 0; i < 32; i++) {
        if (a & (0x80000000u >> i)) p ^= b;
        b = (b >> 1) ^ ((b & 1u) ? BGZF_POLY : 0u);
    }
    return p;
}

// x^(8 n) modulo the polynomial: appending n zero bytes to a message multiplies its CRC register by this
__device__ __forceinline__ uint32_t bgzf_x8n(uint32_t n) {
    uint32_t r = 0x80000000u, sq = 1u << 23;   // x^0, x^8
    for (; n; n >>= 1) {
        if (n & 1u) r = bgzf_mulmod(r, sq);
        sq = bgzf_mulmod(sq, sq);
    }
    return r;
}

// entry b of the byte-at-a-time CRC table
__device__ __forceinline__ uint32_t bgzf_crc_entry(uint32_t b) {
    for (int k = 0; k < 8; k++) b = (b >> 1) ^ ((b & 1u) ? BGZF_POLY : 0u);
    return b;
}
