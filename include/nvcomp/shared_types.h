/*
 * nvcomp/shared_types.h -- status and element-type enums shared by every
 * batched codec of the H100-native nvCOMP-compatible library.
 *
 * Boundary evidence (the reference ships no headers; values are pinned by its
 * call sites): nvcompSuccess / nvcompErrorBadChecksum
 * (examples/high_level_quickstart_example.cpp:314), nvcompErrorAlignment
 * (CHANGELOG.md:16); nvcompType_t numeric values from the error texts
 * "0-5 or 255 (CHAR, UCHAR, SHORT, USHORT, INT, UINT, or BITS)"
 * (benchmarks/benchmark_lz4_chunked.cu:69-70) and "0-7 (... LONGLONG, or
 * ULONGLONG)" (benchmarks/benchmark_cascaded_chunked.cu:109-110).
 */
#ifndef NVCOMP_SHARED_TYPES_H
#define NVCOMP_SHARED_TYPES_H

#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#define NVCOMP_MAJOR_VERSION 3
#define NVCOMP_MINOR_VERSION 0
#define NVCOMP_PATCH_VERSION 3

#ifdef __cplusplus
extern "C" {
#endif

typedef enum nvcompStatus_t
{
  nvcompSuccess = 0,
  nvcompErrorInvalidValue = 10,
  nvcompErrorNotSupported = 11,
  nvcompErrorCannotDecompress = 12,
  nvcompErrorBadChecksum = 13,
  nvcompErrorCannotVerifyChecksums = 14,
  nvcompErrorOutputBufferTooSmall = 15,
  nvcompErrorWrongHeaderLength = 16,
  nvcompErrorAlignment = 17,
  nvcompErrorChunkSizeTooLarge = 18,
  nvcompErrorCudaError = 1000,
  nvcompErrorInternal = 10000
} nvcompStatus_t;

typedef enum nvcompType_t
{
  NVCOMP_TYPE_CHAR = 0,      /* 1B */
  NVCOMP_TYPE_UCHAR = 1,     /* 1B */
  NVCOMP_TYPE_SHORT = 2,     /* 2B */
  NVCOMP_TYPE_USHORT = 3,    /* 2B */
  NVCOMP_TYPE_INT = 4,       /* 4B */
  NVCOMP_TYPE_UINT = 5,      /* 4B */
  NVCOMP_TYPE_LONGLONG = 6,  /* 8B */
  NVCOMP_TYPE_ULONGLONG = 7, /* 8B */
  NVCOMP_TYPE_BITS = 0xff    /* 1b */
} nvcompType_t;

#ifdef __cplusplus
}
#endif

#endif
