// Numeric contract of the library: operation codes, flags, data types, error
// bits.  Values that cross the host/device boundary inside a call descriptor
// are kept numerically identical to the reference so that descriptors, error
// words and test expectations carry over:
//   operation / cfgFunc      driver/xrt/include/accl/constants.hpp:179-210
//   reduceFunction           :218-221      dataType   :256-273
//   stream/host/compression flags :279-326 errorCode  :355-384
// New on H100: bfloat16 and the two fp8 formats (wire/"compressed" types for
// block-scaled transfers), and NVLink-era transport names.
#pragma once
#include <cstddef>
#include <cstdint>
#include <string>

#include "accl/common.hpp"

namespace accl {

using addr_t = uint64_t;
using val_t = uint32_t;
using communicatorId = unsigned int;
using ACCLRequest = long long; // opaque request id handed to the user

constexpr unsigned int TAG_ANY = 0xFFFFFFFFu;
constexpr communicatorId GLOBAL_COMM = 0;
// stream ids below this are reserved (the reference burns 0-8 on switch ports)
constexpr unsigned int STREAM_ID_MIN = 9;
constexpr unsigned int STREAM_ID_MAX = 246;
constexpr int ACCL_MAX_RANKS = 16;       // one NVSwitch domain (8 on HGX H100)
constexpr int ACCL_MAX_COMMUNICATORS = 8;

enum class operation : uint32_t {
  config = 0,
  copy = 1,
  combine = 2,
  send = 3,
  recv = 4,
  bcast = 5,
  scatter = 6,
  gather = 7,
  reduce = 8,
  allgather = 9,
  allreduce = 10,
  reduce_scatter = 11,
  barrier = 12,
  alltoall = 13,
  alltoallv = 14, // uneven all-to-all, per-peer counts read from device memory (beyond the reference)
  nop = 255
};
const char *operation_name(operation op);

enum class cfgFunc : uint32_t {
  reset_periph = 0,
  enable_pkt = 1,
  set_timeout = 2,
  set_max_eager_msg_size = 3,
  set_max_rendezvous_msg_size = 4
};

enum class reduceFunction : uint32_t { SUM = 0, MAX = 1 };

enum class dataType : uint32_t {
  none = 0,
  int8 = 1,
  float16 = 2,
  float32 = 3,
  float64 = 4,
  int32 = 5,
  int64 = 6,
  bfloat16 = 7,
  float8_e4m3 = 8,
  float8_e5m2 = 9
};
constexpr int ACCL_NUM_DTYPES = 10;

ACCL_HD unsigned int dtype_bits(dataType t) {
  switch (t) {
  case dataType::int8: return 8;
  case dataType::float16: return 16;
  case dataType::float32: return 32;
  case dataType::float64: return 64;
  case dataType::int32: return 32;
  case dataType::int64: return 64;
  case dataType::bfloat16: return 16;
  case dataType::float8_e4m3: return 8;
  case dataType::float8_e5m2: return 8;
  default: return 0;
  }
}
ACCL_HD unsigned int dtype_bytes(dataType t) { return dtype_bits(t) / 8; }
const char *dtype_name(dataType t);

enum class streamFlags : uint32_t { NO_STREAM = 0, OP0_STREAM = 1, RES_STREAM = 2 };
enum class hostFlags : uint32_t { NO_HOST = 0, OP0_HOST = 1, OP1_HOST = 2, RES_HOST = 4 };
enum class compressionFlags : uint32_t {
  NO_COMPRESSION = 0,
  OP0_COMPRESSED = 1,
  OP1_COMPRESSED = 2,
  RES_COMPRESSED = 4,
  ETH_COMPRESSED = 8 // "wire" compressed: the NVLink payload uses the compressed type
};

#define ACCL_FLAG_OPS(E)                                                                         \
  constexpr E operator|(E a, E b) { return static_cast<E>(static_cast<uint32_t>(a) | static_cast<uint32_t>(b)); } \
  constexpr E operator&(E a, E b) { return static_cast<E>(static_cast<uint32_t>(a) & static_cast<uint32_t>(b)); } \
  inline E &operator|=(E &a, E b) { return a = a | b; }                                          \
  constexpr bool any(E a) { return static_cast<uint32_t>(a) != 0; }
ACCL_FLAG_OPS(streamFlags)
ACCL_FLAG_OPS(hostFlags)
ACCL_FLAG_OPS(compressionFlags)
#undef ACCL_FLAG_OPS

// Which fabric moves the bytes.  The reference selects UDP/TCP/RDMA POEs at
// bitstream build time (constants.hpp:334-338); here the choice is between
// the NVLink backend and the two emulator wires.
enum class networkProtocol : uint32_t { NVLINK = 0, EMU_INPROC = 1, EMU_SOCKET = 2 };

enum class deviceType : uint32_t { emulator = 0, cuda = 1 };

// One bit per failure cause, OR-ed into the per-call return word.
enum errorCode : uint32_t {
  COLLECTIVE_OP_SUCCESS = 0,
  DMA_MISMATCH_ERROR = 1u << 0,
  DMA_INTERNAL_ERROR = 1u << 1,
  DMA_DECODE_ERROR = 1u << 2,
  DMA_SLAVE_ERROR = 1u << 3,
  DMA_NOT_OKAY_ERROR = 1u << 4,
  DMA_NOT_END_OF_PACKET_ERROR = 1u << 5,
  DMA_NOT_EXPECTED_BTT_ERROR = 1u << 6,
  DMA_TIMEOUT_ERROR = 1u << 7,
  CONFIG_SWITCH_ERROR = 1u << 8,
  DEQUEUE_BUFFER_TIMEOUT_ERROR = 1u << 9,
  DEQUEUE_BUFFER_SPARE_BUFFER_STATUS_ERROR = 1u << 10,
  RECEIVE_TIMEOUT_ERROR = 1u << 11,
  DEQUEUE_BUFFER_SPARE_BUFFER_DMATAG_MISMATCH = 1u << 12,
  DEQUEUE_BUFFER_SPARE_BUFFER_INDEX_ERROR = 1u << 13,
  COLLECTIVE_NOT_IMPLEMENTED = 1u << 14,
  RECEIVE_OFFCHIP_SPARE_BUFF_ID_NOT_VALID = 1u << 15,
  EAGER_THRESHOLD_INVALID = 1u << 16,
  RENDEZVOUS_THRESHOLD_INVALID = 1u << 17,
  DMA_SIZE_ERROR = 1u << 18,
  ARITH_ERROR = 1u << 19,
  PACK_TIMEOUT_STS_ERROR = 1u << 20,
  PACK_SEQ_NUMBER_ERROR = 1u << 21,
  COMPRESSION_ERROR = 1u << 22,
  KRNL_TIMEOUT_STS_ERROR = 1u << 23,
  KRNL_STS_COUNT_ERROR = 1u << 24,
  SEGMENTER_EXPECTED_BTT_ERROR = 1u << 25,
  DMA_TAG_MISMATCH_ERROR = 1u << 26,
  // internal: the call could not make progress yet and was parked
  NOT_READY_ERROR = 1u << 31
};
constexpr int ACCL_NUM_ERROR_BITS = 27;
const char *error_code_to_string(errorCode bit);
// decode an OR of error bits into "NAME | NAME | ..."
std::string error_word_to_string(uint32_t word);

// Capability word reported by the backend (the reference's HWID register,
// accl.cpp:1050-1064): which optional datapaths exist.
enum capability : uint32_t {
  CAP_DMA = 1u << 0,
  CAP_ARITH = 1u << 1,
  CAP_COMPRESSION = 1u << 2,
  CAP_STREAMS = 1u << 3,      // device-side producer/consumer streams
  CAP_RENDEZVOUS = 1u << 4,
  CAP_NVLS_MULTICAST = 1u << 5, // in-switch reduce / broadcast available
  CAP_PERSISTENT_ENGINE = 1u << 6,
  CAP_FP8 = 1u << 7,
  CAP_TCGEN05 = 1u << 8
};

} // namespace accl
