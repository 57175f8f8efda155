// crc32.cuh -- standard CRC-32 (IEEE 802.3, reflected polynomial 0xEDB88320, the zlib value): the internal interface
// of crc32.cu used by the high-level interface for its whole-buffer checksums.  The warp routine that hashes one span
// (crc0_warp + crc_finish) and its table entries live in nvcomp/device/detail/crc32.cuh, shared with the Gzip decoder
// and the device API of nvcomp/device/gzip.cuh; this file re-exports them into namespace b200.
#pragma once

#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "common.cuh"
#include "nvcomp/device/detail/crc32.cuh"

namespace b200 {

using nvcomp::device::crc::detail::kCrcPoly;
using nvcomp::device::crc::detail::crc_mulmod;
using nvcomp::device::crc::detail::crc_table_entry;
using nvcomp::device::crc::detail::crc_x2n_entry;
using nvcomp::device::crc::detail::crc_x8n;
using nvcomp::device::crc::detail::crc_bytes;
using nvcomp::device::crc::detail::crc0_warp;
using nvcomp::device::crc::detail::crc_finish;

constexpr size_t kCrcPiece = 65536;            // bytes hashed by one warp

// u32 words of scratch crc32_buffer_async needs for a buffer of at most max_bytes
size_t crc_scratch_words(size_t max_bytes);

// *result = CRC-32 of data[0, n) where n = n_host, or (*len_dev - skip) when len_dev != nullptr (a length
// only the device knows, e.g. the compressed size); max_bytes bounds n and sizes the launch.  Asynchronous.
cudaError_t crc32_buffer_async(const uint8_t* data, size_t n_host, const unsigned long long* len_dev, size_t skip,
                               size_t max_bytes, uint32_t* piece_scratch, uint32_t* result, cudaStream_t stream);

}  // namespace b200
