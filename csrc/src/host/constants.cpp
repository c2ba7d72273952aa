#include "accl/constants.hpp"

namespace accl {

const char *operation_name(operation op) {
  switch (op) {
  case operation::config: return "config";
  case operation::copy: return "copy";
  case operation::combine: return "combine";
  case operation::send: return "send";
  case operation::recv: return "recv";
  case operation::bcast: return "bcast";
  case operation::scatter: return "scatter";
  case operation::gather: return "gather";
  case operation::reduce: return "reduce";
  case operation::allgather: return "allgather";
  case operation::allreduce: return "allreduce";
  case operation::reduce_scatter: return "reduce_scatter";
  case operation::barrier: return "barrier";
  case operation::alltoall: return "alltoall";
  case operation::alltoallv: return "alltoallv";
  case operation::nop: return "nop";
  }
  return "unknown";
}

const char *dtype_name(dataType t) {
  switch (t) {
  case dataType::none: return "none";
  case dataType::int8: return "int8";
  case dataType::float16: return "float16";
  case dataType::float32: return "float32";
  case dataType::float64: return "float64";
  case dataType::int32: return "int32";
  case dataType::int64: return "int64";
  case dataType::bfloat16: return "bfloat16";
  case dataType::float8_e4m3: return "float8_e4m3";
  case dataType::float8_e5m2: return "float8_e5m2";
  }
  return "invalid";
}

const char *error_code_to_string(errorCode bit) {
  switch (bit) {
  case COLLECTIVE_OP_SUCCESS: return "COLLECTIVE_OP_SUCCESS";
  case DMA_MISMATCH_ERROR: return "DMA_MISMATCH_ERROR";
  case DMA_INTERNAL_ERROR: return "DMA_INTERNAL_ERROR";
  case DMA_DECODE_ERROR: return "DMA_DECODE_ERROR";
  case DMA_SLAVE_ERROR: return "DMA_SLAVE_ERROR";
  case DMA_NOT_OKAY_ERROR: return "DMA_NOT_OKAY_ERROR";
  case DMA_NOT_END_OF_PACKET_ERROR: return "DMA_NOT_END_OF_PACKET_ERROR";
  case DMA_NOT_EXPECTED_BTT_ERROR: return "DMA_NOT_EXPECTED_BTT_ERROR";
  case DMA_TIMEOUT_ERROR: return "DMA_TIMEOUT_ERROR";
  case CONFIG_SWITCH_ERROR: return "CONFIG_SWITCH_ERROR";
  case DEQUEUE_BUFFER_TIMEOUT_ERROR: return "DEQUEUE_BUFFER_TIMEOUT_ERROR";
  case DEQUEUE_BUFFER_SPARE_BUFFER_STATUS_ERROR: return "DEQUEUE_BUFFER_SPARE_BUFFER_STATUS_ERROR";
  case RECEIVE_TIMEOUT_ERROR: return "RECEIVE_TIMEOUT_ERROR";
  case DEQUEUE_BUFFER_SPARE_BUFFER_DMATAG_MISMATCH: return "DEQUEUE_BUFFER_SPARE_BUFFER_DMATAG_MISMATCH";
  case DEQUEUE_BUFFER_SPARE_BUFFER_INDEX_ERROR: return "DEQUEUE_BUFFER_SPARE_BUFFER_INDEX_ERROR";
  case COLLECTIVE_NOT_IMPLEMENTED: return "COLLECTIVE_NOT_IMPLEMENTED";
  case RECEIVE_OFFCHIP_SPARE_BUFF_ID_NOT_VALID: return "RECEIVE_OFFCHIP_SPARE_BUFF_ID_NOT_VALID";
  case EAGER_THRESHOLD_INVALID: return "EAGER_THRESHOLD_INVALID";
  case RENDEZVOUS_THRESHOLD_INVALID: return "RENDEZVOUS_THRESHOLD_INVALID";
  case DMA_SIZE_ERROR: return "DMA_SIZE_ERROR";
  case ARITH_ERROR: return "ARITH_ERROR";
  case PACK_TIMEOUT_STS_ERROR: return "PACK_TIMEOUT_STS_ERROR";
  case PACK_SEQ_NUMBER_ERROR: return "PACK_SEQ_NUMBER_ERROR";
  case COMPRESSION_ERROR: return "COMPRESSION_ERROR";
  case KRNL_TIMEOUT_STS_ERROR: return "KRNL_TIMEOUT_STS_ERROR";
  case KRNL_STS_COUNT_ERROR: return "KRNL_STS_COUNT_ERROR";
  case SEGMENTER_EXPECTED_BTT_ERROR: return "SEGMENTER_EXPECTED_BTT_ERROR";
  case DMA_TAG_MISMATCH_ERROR: return "DMA_TAG_MISMATCH_ERROR";
  case NOT_READY_ERROR: return "NOT_READY_ERROR";
  }
  return "UNKNOWN_ERROR";
}

std::string error_word_to_string(uint32_t word) {
  if (word == 0) return "COLLECTIVE_OP_SUCCESS";
  std::string s;
  for (int b = 0; b < 32; ++b) {
    if (!(word & (1u << b))) continue;
    if (!s.empty()) s += " | ";
    s += error_code_to_string(static_cast<errorCode>(1u << b));
  }
  return s;
}

} // namespace accl
