// RotaryMulQueryOp (op type "RotaryMulQuery") — forwarder to b2_rotary / b2_rotary_table.
// Reference: csrc/core/operator/general/rotary_multiquery/rotary_mulquery_op.cpp (ChatGLM2 / ChatGLM3 / GLM-4 graphs,
// chatglm_v2.py): the rotary of the q and k heads of the fused QKV activation, V passed through.  Supported:
//   rotary_type 0 (base): NeoX rotate-half over the whole head at rotary_base (b2_rotary, bf16);
//   rotary_type 3 (half_inner): the interleaved pairs (2i, 2i + 1) over the first head / 2 dims, frequencies
//     invfreq_type 1: base^(-2i / (head / 2)) / rope_ratio, or 2: (base rope_ratio)^(-2i / (head / 2)), built once at Init
//     as an fp32 device table (b2_rotary_table with B2_ROPE_INTERLEAVED, bf16 or fp16).
// Other rotary_type / invfreq_type values are refused at Init (ALLSPARK_PARAM_ERROR, the status of an unsupported
// configuration).  Positions: gen_ctx->step of each sequence, like the reference's step_list.
#pragma once
#include <memory>
#include <vector>

#include "operator.h"

namespace allspark {

class RotaryMulQueryOp : public AsOperator {
 public:
  using AsOperator::AsOperator;
  AsStatus Init(const OperatorProto& op_proto, const DeviceContext& ctx, const TensorMap& weights_map, TensorMap* tensor_map) override;
  AsStatus Reshape(RuntimeContext* runtime_ctx) override;
  AsStatus Forward(RuntimeContext* runtime_ctx) override;

 private:
  int num_heads_ = 0, groups_ = 0, head_dim_ = 0, rows_ = 0, rotary_type_ = 0, invfreq_type_ = 0;
  float base_ = 10000.f, rope_ratio_ = 1.f;
  DataType dtype_ = DataType::BFLOAT16;
  std::unique_ptr<AsTensor> inv_freq_, pos_;  // fp32 [head / 4] (rotary_type 3); int32 [rows]
  std::vector<int32_t> pos_h_;
};

}  // namespace allspark
