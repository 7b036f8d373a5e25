// QKLayerNormNoBetaOp (op type "QKLayerNormNoBeta") — forwarder to b2_qk_rmsnorm.
// Reference: csrc/core/operator/general/qk_layernorm_nobeta/qk_layernorm_nobeta_op.cpp (Qwen3, qwen_v30.py): per-head
// RMSNorm of the q and k heads of the fused QKV activation before Rotary, V passed through.  The reference builds host
// arrays of per-head row pointers and copies them to the device on every call; here one kernel walks [rows, ld] directly,
// stream-ordered and CUDA-graph replayable.
#pragma once
#include "operator.h"

namespace allspark {

class QKLayerNormNoBetaOp : public AsOperator {
 public:
  using AsOperator::AsOperator;
  AsStatus Init(const OperatorProto& op_proto, const DeviceContext& ctx, const TensorMap& weights_map, TensorMap* tensor_map) override;
  AsStatus Reshape(RuntimeContext* runtime_ctx) override;
  AsStatus Reshape() override { return Reshape(nullptr); }
  AsStatus Forward(RuntimeContext* runtime_ctx) override;
  AsStatus Forward() override { return Forward(nullptr); }

 private:
  int head_dim_ = 0, num_heads_ = 0, groups_ = 0, rows_ = 0;
  float eps_ = 1e-6f;
  DataType dtype_ = DataType::BFLOAT16;
};

}  // namespace allspark
