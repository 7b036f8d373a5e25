#include "qk_layernorm_op.h"

namespace allspark {

// Weights [q_gamma, k_gamma] ([head_dim] each); attributes eps, num_heads, multi_query_group_num, the head counts divided
// by the number of TP ranks like qk_layernorm_nobeta_op.cpp:110-113 (a group count of 1 is kept: one kv head replicated).
AsStatus QKLayerNormNoBetaOp::Init(const OperatorProto& op_proto, const DeviceContext& ctx, const TensorMap& weights_map,
                                   TensorMap* tensor_map) {
  AS_CHECK_STATUS(AsOperator::Init(op_proto, ctx, weights_map, tensor_map));
  if (weights_.size() != 2) {
    AS_LOG_ERROR("QKLayerNormNoBeta: 2 weights [q_gamma, k_gamma] expected, got %zu\n", weights_.size());
    return AsStatus::ALLSPARK_PARAM_ERROR;
  }
  head_dim_ = (int)weights_[0]->GetShape()[0];
  dtype_ = weights_[0]->GetDataType();
  if (weights_[1]->GetShape()[0] != head_dim_ || weights_[1]->GetDataType() != dtype_) {
    AS_LOG_ERROR("QKLayerNormNoBeta: q_gamma and k_gamma differ in shape or type\n");
    return AsStatus::ALLSPARK_PARAM_ERROR;
  }
  auto& attr = op_proto.attr();
  for (const char* k : {"eps", "num_heads", "multi_query_group_num"})
    if (!attr.count(k)) {
      AS_LOG_ERROR("QKLayerNormNoBeta: attribute %s missing\n", k);
      return AsStatus::ALLSPARK_PARAM_ERROR;
    }
  eps_ = *(const float*)attr.at("eps").c_str();
  num_heads_ = *(const int*)attr.at("num_heads").c_str();
  groups_ = *(const int*)attr.at("multi_query_group_num").c_str();
  const int nranks = ctx.GetNranks() > 0 ? ctx.GetNranks() : 1;
  num_heads_ /= nranks;
  if (groups_ != 1) groups_ /= nranks;
  tensor_map_->at(out_names_[0])->SetDataType(dtype_);
  return AsStatus::ALLSPARK_SUCCESS;
}

// input and output [batch, 1, (nH + 2 nG) * head_dim]
AsStatus QKLayerNormNoBetaOp::Reshape(RuntimeContext*) {
  Shape s = tensor_map_->at(in_names_[0])->GetShape();
  const int64_t width = (int64_t)(num_heads_ + 2 * groups_) * head_dim_;
  if (s.Size() < 1 || s[-1] != width) {
    AS_LOG_ERROR("QKLayerNormNoBeta: input rows of %lld values, (num_heads + 2 groups) * head_dim = %lld\n",
                 (long long)(s.Size() ? s[-1] : 0), (long long)width);
    return AsStatus::ALLSPARK_PARAM_ERROR;
  }
  rows_ = (int)(s.Count() / width);
  return tensor_map_->at(out_names_[0])->SetShape(std::move(s));
}

AsStatus QKLayerNormNoBetaOp::Forward(RuntimeContext*) {
  const CUDAContext* cc = static_cast<const CUDAContext*>(ctx_);
  b2_qk_norm norm{weights_[0]->GetDataPtr(), weights_[1]->GetDataPtr(), eps_, 0};
  return FromB2(b2_qk_rmsnorm(tensor_map_->at(out_names_[0])->GetDataPtr(), tensor_map_->at(in_names_[0])->GetDataPtr(), rows_,
                              (int64_t)(num_heads_ + 2 * groups_) * head_dim_, num_heads_, groups_, head_dim_, &norm,
                              (int)dtype_, cc->GetStream()));
}

REGISTER_OP(QKLayerNormNoBeta, CUDA, QKLayerNormNoBetaOp)

}  // namespace allspark
