#include "rotary_mulquery_op.h"

#include <cmath>

namespace allspark {

namespace {
template <typename T>
T attr_or(const OperatorProto& p, const char* k, T dflt) {
  auto& a = p.attr();
  return a.count(k) ? *(const T*)a.at(k).c_str() : dflt;
}
}  // namespace

// Attributes as the reference's converter sets them (chatglm_v2.py: num_heads, multi_query_group_num, hidden_size,
// rotary_type, rope_ratio, invfreq_type; rotary_base, default 10000).  Head counts are the whole model's and are divided by
// the number of TP ranks (a group count of 1 is kept: one kv head replicated), like QKLayerNormNoBeta.
AsStatus RotaryMulQueryOp::Init(const OperatorProto& op_proto, const DeviceContext& ctx, const TensorMap& weights_map,
                                TensorMap* tensor_map) {
  AS_CHECK_STATUS(AsOperator::Init(op_proto, ctx, weights_map, tensor_map));
  auto& attr = op_proto.attr();
  for (const char* k : {"num_heads", "multi_query_group_num", "hidden_size"})
    if (!attr.count(k)) {
      AS_LOG_ERROR("RotaryMulQuery: attribute %s missing\n", k);
      return AsStatus::ALLSPARK_PARAM_ERROR;
    }
  num_heads_ = *(const int*)attr.at("num_heads").c_str();
  groups_ = *(const int*)attr.at("multi_query_group_num").c_str();
  const int hidden = *(const int*)attr.at("hidden_size").c_str();
  rotary_type_ = attr_or<int>(op_proto, "rotary_type", 0);
  invfreq_type_ = attr_or<int>(op_proto, "invfreq_type", 0);
  rope_ratio_ = attr_or<float>(op_proto, "rope_ratio", 1.f);
  base_ = attr_or<float>(op_proto, "rotary_base", 10000.f);
  if (num_heads_ <= 0 || groups_ <= 0 || hidden % num_heads_) {
    AS_LOG_ERROR("RotaryMulQuery: num_heads %d, multi_query_group_num %d, hidden_size %d\n", num_heads_, groups_, hidden);
    return AsStatus::ALLSPARK_PARAM_ERROR;
  }
  head_dim_ = hidden / num_heads_;
  const int nranks = ctx.GetNranks() > 0 ? ctx.GetNranks() : 1;
  num_heads_ /= nranks;
  if (groups_ != 1) groups_ /= nranks;
  dtype_ = tensor_map_->at(in_names_[0])->GetDataType();
  const bool half_inner = rotary_type_ == 3 && (invfreq_type_ == 1 || invfreq_type_ == 2);
  if (!(rotary_type_ == 0 && dtype_ == DataType::BFLOAT16) && !half_inner) {
    AS_LOG_ERROR("RotaryMulQuery: rotary_type %d / invfreq_type %d (dtype %d) not supported\n", rotary_type_, invfreq_type_,
                 (int)dtype_);
    return AsStatus::ALLSPARK_PARAM_ERROR;
  }
  if (half_inner) {  // the fp32 frequencies of the first head / 2 dims, computed in double and rounded once
    const int rd = head_dim_ / 2;
    std::vector<float> inv(rd / 2);
    for (int i = 0; i < rd / 2; ++i) {
      const double e = -2.0 * i / rd;
      inv[i] = (float)(invfreq_type_ == 1 ? std::pow((double)base_, e) / (double)rope_ratio_
                                           : std::pow((double)base_ * (double)rope_ratio_, e));
    }
    inv_freq_ = std::make_unique<AsTensor>("rotary_inv_freq", DeviceType::CUDA, DataType::FLOAT32, DataMode::DENSE,
                                           Shape{(int64_t)inv.size()});
    inv_freq_->CopyDataFrom(inv.data(), inv.size() * sizeof(float), DeviceType::CPU);
  }
  tensor_map_->at(out_names_[0])->SetDataType(dtype_);
  return AsStatus::ALLSPARK_SUCCESS;
}

// input and output [batch, 1, (nH + 2 nG) * head_dim]
AsStatus RotaryMulQueryOp::Reshape(RuntimeContext*) {
  Shape s = tensor_map_->at(in_names_[0])->GetShape();
  const int64_t width = (int64_t)(num_heads_ + 2 * groups_) * head_dim_;
  if (s.Size() < 1 || s[-1] != width) {
    AS_LOG_ERROR("RotaryMulQuery: input rows of %lld values, (num_heads + 2 groups) * head_dim = %lld\n",
                 (long long)(s.Size() ? s[-1] : 0), (long long)width);
    return AsStatus::ALLSPARK_PARAM_ERROR;
  }
  rows_ = (int)(s.Count() / width);
  if (!pos_ || pos_->GetShape()[0] < rows_)
    pos_ = std::make_unique<AsTensor>("rotary_pos", DeviceType::CUDA, DataType::INT32, DataMode::DENSE, Shape{rows_});
  return tensor_map_->at(out_names_[0])->SetShape(std::move(s));
}

AsStatus RotaryMulQueryOp::Forward(RuntimeContext* runtime_ctx) {
  if (!runtime_ctx || runtime_ctx->GetGenCtxListSize() < rows_) {
    AS_LOG_ERROR("RotaryMulQuery: the positions come from one generate context per row\n");
    return AsStatus::ALLSPARK_PARAM_ERROR;
  }
  const CUDAContext* cc = static_cast<const CUDAContext*>(ctx_);
  cudaStream_t stream = cc->GetStream();
  pos_h_.resize(rows_);
  for (int b = 0; b < rows_; ++b) pos_h_[b] = runtime_ctx->GetGenCtx(b)->step;
  // pageable source: the copy has read pos_h_ when the call returns
  if (cudaMemcpyAsync(pos_->GetDataPtr(), pos_h_.data(), rows_ * sizeof(int32_t), cudaMemcpyHostToDevice, stream) != cudaSuccess)
    return AsStatus::ALLSPARK_RUNTIME_ERROR;
  AsTensor* in = tensor_map_->at(in_names_[0]).get();
  AsTensor* out = tensor_map_->at(out_names_[0]).get();
  if (out->GetDataPtr() != in->GetDataPtr() &&
      cudaMemcpyAsync(out->GetDataPtr(), in->GetDataPtr(), in->GetSizeInByte(), cudaMemcpyDeviceToDevice, stream) != cudaSuccess)
    return AsStatus::ALLSPARK_RUNTIME_ERROR;
  const int32_t* pos = (const int32_t*)pos_->GetDataPtr();
  if (rotary_type_ == 0) {
    b2_rope_cfg rope{base_, head_dim_, B2_ROPE_NEOX};
    return FromB2(b2_rotary(out->GetDataPtr(), pos, rows_, num_heads_, groups_, head_dim_, &rope, stream));
  }
  b2_rope_cfg rope{0.f, head_dim_ / 2, B2_ROPE_INTERLEAVED};
  b2_rope_table table{(const float*)inv_freq_->GetDataPtr(), 0, 1.f, 0};
  return FromB2(b2_rotary_table(out->GetDataPtr(), pos, rows_, num_heads_, groups_, head_dim_, &rope, &table, (int)dtype_, stream));
}

REGISTER_OP(RotaryMulQuery, CUDA, RotaryMulQueryOp)

}  // namespace allspark
