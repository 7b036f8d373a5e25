// C entry points that drive the allspark-shaped operators the way the reference's TestOpUtil does
// (tests/cpp/operator/test_operator_utils.h:24-112, operator_gemm_lowp_test.cpp:650-725): fabricate an OperatorProto,
// a DeviceContext and a TensorMap with "workspace", then InitV2 -> Reshape -> Forward.  Used by tests/test_host_ops_gpu.py.
#include <cstring>
#include <memory>
#include <vector>

#include "allreduce_op.h"
#include "gemm_lowp_gpu.h"
#include "qk_layernorm_op.h"
#include "rotary_mulquery_op.h"
#include "span_attn_op_cuda.h"

using namespace allspark;

// the 16-bit model dtype the test entry points below build their tensors with (BFLOAT16 unless as_test_set_dtype says FLOAT16)
static allspark::DataType g_test_ft = allspark::DataType::BFLOAT16;

extern "C" {
int as_test_set_dtype(int dt) {
  if (dt != (int)allspark::DataType::BFLOAT16 && dt != (int)allspark::DataType::FLOAT16) return -1;
  g_test_ft = (allspark::DataType)dt;
  return 0;
}


int as_test_registered(const char* op_type) {
  try {
    auto c = OpFactory::getInstance().GetOperator({op_type, DeviceType::CUDA});
    return c ? 1 : 0;
  } catch (...) {
    return 0;
  }
}

// op_type: "GemmA16W4" | "GemmA16W8" | "Gemm".  Host buffers in the reference layouts; C_host receives [M, N] bf16.
static int run_gemm(const char* op_type, int M, int N, int K, int group_size, int activation, float alpha, const void* A_host,
                    const void* w_host, int w_dtype, const void* scales_host, const void* zeros_host, const void* bias_host,
                    const void* residual_host, int binary_type, void* C_host) {
  try {
    CUDAContext ctx;
    ctx.SetDtype(g_test_ft);
    ctx.SetModelMaxBatch(M);
    TensorMap tensors, weights, weights_buffer;
    const std::string t = op_type;
    const bool quant = t != "Gemm";
    const int wbits = t == "GemmA16W4" ? 4 : (t == "GemmA16W8" ? 8 : 16);
    auto add = [&](TensorMap& m, const std::string& name, DataType dt, Shape s, const void* src) {
      auto ten = std::make_shared<AsTensor>(name, DeviceType::CUDA, dt, DataMode::DENSE, s);
      if (src) ten->CopyDataFrom(src, ten->GetSizeInByte(), DeviceType::CPU);
      m[name] = ten;
    };
    add(tensors, "input", g_test_ft, Shape{1, M, K}, A_host);
    tensors["workspace"] = std::make_shared<AsTensor>("workspace", DeviceType::CUDA, DataType::INT8, DataMode::DENSE, Shape{0});
    const int G = group_size == -1 ? 1 : (K + group_size - 1) / group_size;
    if (wbits == 4) add(weights, "weight", (DataType)w_dtype, Shape{K, (N + 1) / 2}, w_host);
    else if (wbits == 8) add(weights, "weight", (DataType)w_dtype, Shape{K, N}, w_host);
    else add(weights, "weight", g_test_ft, Shape{K, N}, w_host);
    OperatorProto proto;
    proto.op_type_ = t; proto.op_name_ = "test_" + t;
    proto.inputs_.push_back({"input"}); proto.outputs_.push_back({"output"});
    proto.weights_.push_back({"weight"});
    if (residual_host) {  // do_binary_add_fused graphs: Gemm(x, residual) with binary_type ADD (qwen_v15.py:280-286)
      add(tensors, "residual", g_test_ft, Shape{1, M, N}, residual_host);
      proto.inputs_.push_back({"residual"});
    }
    if (binary_type) proto.SetAttr<int>("binary_type", binary_type);
    if (quant) {
      add(weights, "scales", g_test_ft, Shape{G, N}, scales_host);
      add(weights, "zeros", g_test_ft, Shape{G, N}, zeros_host);
      proto.weights_.push_back({"scales"}); proto.weights_.push_back({"zeros"});
      if (group_size != -1) proto.SetAttr<int>("GroupSize", group_size);
    }
    if (bias_host) {
      add(weights, "bias", g_test_ft, Shape{N}, bias_host);
      proto.weights_.push_back({"bias"});
    }
    proto.SetAttr<float>("alpha", alpha);
    proto.SetAttr<bool>("is_pooler", false);
    if (activation) proto.SetAttr<int>("activation", activation);
    auto op = OpFactory::getInstance().GetOperator({t, DeviceType::CUDA})();
    AsStatus st = op->InitV2(proto, ctx, weights, weights_buffer, &tensors, nullptr);
    if (st != AsStatus::ALLSPARK_SUCCESS) return (int)st;
    st = op->Reshape();
    if (st != AsStatus::ALLSPARK_SUCCESS) return (int)st;
    st = op->Forward();
    if (st != AsStatus::ALLSPARK_SUCCESS) return (int)st;
    ctx.Synchronize();
    auto out = tensors["output"];
    if (out->GetShape().Count() != (int64_t)M * N) return -2;
    out->CopyDataTo(C_host, out->GetSizeInByte(), DeviceType::CPU);
    return cudaGetLastError() == cudaSuccess ? 0 : -3;
  } catch (const std::exception& e) {
    AS_LOG_ERROR("as_test_gemm: %s", e.what());
    return -1;
  }
}

int as_test_gemm(const char* op_type, int M, int N, int K, int group_size, int activation, float alpha, const void* A_host,
                 const void* w_host, int w_dtype, const void* scales_host, const void* zeros_host, const void* bias_host,
                 void* C_host) {
  return run_gemm(op_type, M, N, K, group_size, activation, alpha, A_host, w_host, w_dtype, scales_host, zeros_host, bias_host,
                  nullptr, 0, C_host);
}

int as_test_gemm_binary(const char* op_type, int M, int N, int K, int group_size, int activation, float alpha, const void* A_host,
                        const void* w_host, int w_dtype, const void* scales_host, const void* zeros_host, const void* bias_host,
                        const void* residual_host, int binary_type, void* C_host) {
  return run_gemm(op_type, M, N, K, group_size, activation, alpha, A_host, w_host, w_dtype, scales_host, zeros_host, bias_host,
                  residual_host, binary_type, C_host);
}

// nranks AllReduce ops (one context / stream / communicator per "rank", all on the current device, wired through
// b2_comm_connect_pointers) reduce nranks host vectors of `count` bf16; every rank's result is copied to out_all[r].
int as_test_allreduce(int nranks, int64_t count, const void* in_all, void* out_all) {
  try {
    std::vector<b2_comm_t> comms(nranks, nullptr);
    std::vector<void*> bufs(nranks, nullptr);
    for (int r = 0; r < nranks; ++r) {
      if (b2_comm_create(&comms[r], r, nranks, (size_t)count * 2) != B2_OK) return -4;
      bufs[r] = b2_comm_local_buffer(comms[r]);
    }
    for (int r = 0; r < nranks; ++r)
      if (b2_comm_connect_pointers(comms[r], bufs.data()) != B2_OK) return -5;
    std::vector<std::unique_ptr<CUDAContext>> ctxs;
    std::vector<std::unique_ptr<TensorMap>> maps;
    std::vector<std::unique_ptr<AsOperator>> ops;
    TensorMap weights;
    for (int r = 0; r < nranks; ++r) {
      ctxs.push_back(std::make_unique<CUDAContext>());
      ctxs[r]->SetDtype(DataType::BFLOAT16);
      ctxs[r]->SetRank(r, nranks);
      ctxs[r]->SetB2Comm(comms[r]);
      maps.push_back(std::make_unique<TensorMap>());
      auto t = std::make_shared<AsTensor>("x", DeviceType::CUDA, DataType::BFLOAT16, DataMode::DENSE, Shape{1, count});
      t->CopyDataFrom((const char*)in_all + (size_t)r * count * 2, (size_t)count * 2, DeviceType::CPU);
      (*maps[r])["x"] = t;
      OperatorProto proto;
      proto.op_type_ = "AllReduce"; proto.op_name_ = "decoder.layer.0.attention.output.dense.allreduce";
      proto.inputs_.push_back({"x"}); proto.outputs_.push_back({"x"});  // in place, like the reference graphs
      ops.push_back(OpFactory::getInstance().GetOperator({"AllReduce", DeviceType::CUDA})());
      TensorMap wb;
      AsStatus st = ops[r]->InitV2(proto, *ctxs[r], weights, wb, maps[r].get(), nullptr);
      if (st != AsStatus::ALLSPARK_SUCCESS) return (int)st;
      st = ops[r]->CallReshape(nullptr);
      if (st != AsStatus::ALLSPARK_SUCCESS) return (int)st;
    }
    cudaDeviceSynchronize();
    for (int it = 0; it < 2; ++it) {  // twice: the second exchange runs on the other buffer parity (input = first result)
      for (int r = 0; r < nranks; ++r) {
        AsStatus st = ops[r]->CallForward(nullptr);
        if (st != AsStatus::ALLSPARK_SUCCESS) return (int)st;
      }
      for (int r = 0; r < nranks; ++r) ctxs[r]->Synchronize();
      if (it == 0)
        for (int r = 0; r < nranks; ++r)
          (*maps[r])["x"]->CopyDataTo((char*)out_all + (size_t)r * count * 2, (size_t)count * 2, DeviceType::CPU);
    }
    int rc = 0;
    for (int r = 0; r < nranks; ++r) {
      if (b2_comm_error(comms[r]) != B2_OK) rc = -6;
      b2_comm_destroy(comms[r]);
    }
    return rc ? rc : (cudaGetLastError() == cudaSuccess ? 0 : -3);
  } catch (const std::exception& e) {
    AS_LOG_ERROR("as_test_allreduce: %s", e.what());
    return -1;
  }
}

// Decode `steps` tokens for `batch` sequences through DecOptMQA: per step op.Alloc + op.Forward with qkv_all[t]
// ([steps][batch][(nH+2nG)*128] bf16); every step's output is written to out_all ([steps][batch][nH*128] bf16).
int as_test_span_attn(int batch, int steps, int n_heads, int n_groups, int span_len, int cache_mode, int max_len, int layers,
                      int layer_id, const void* qkv_all, void* out_all) {
  try {
    CUDAContext ctx;
    ctx.SetDtype(g_test_ft);
    ctx.SetModelMaxBatch(batch);
    ctx.SetModelMaxLength(max_len);
    ctx.SetNumberHeads(n_heads);
    ctx.SetNumberGroups(n_groups);
    ctx.SetSizePerHead(128);
    ctx.SetDecoderLayer(layers);
    auto cc = SpanCacheConfig::Create((AsCacheMode)cache_mode, span_len);
    if (!cc) return (int)AsStatus::ALLSPARK_PARAM_ERROR;
    ctx.SetCacheConfig(cc);
    const size_t span_bytes = CacheUtils::GetSpanSizeInBytes(*cc, g_test_ft, n_groups, 128);
    const int max_spans = (max_len + span_len - 1) / span_len;
    auto pool = std::make_shared<CacheSpanPool>(span_bytes, 2 * batch * layers * max_spans);
    RuntimeContext rt(false);
    for (int b = 0; b < batch; ++b) {
      auto g = std::make_unique<GenerateContext>();
      g->virtual_k_cache = std::make_unique<SpannedVirtualCache>(pool, layers, span_len, max_spans);
      g->virtual_v_cache = std::make_unique<SpannedVirtualCache>(pool, layers, span_len, max_spans);
      rt.PushBackGenCtx(std::move(g));
    }
    const int64_t W = (int64_t)(n_heads + 2 * n_groups) * 128, OW = (int64_t)n_heads * 128;
    TensorMap tensors, weights, weights_buffer;
    tensors["qkv"] = std::make_shared<AsTensor>("qkv", DeviceType::CUDA, g_test_ft, DataMode::DENSE, Shape{batch, 1, W});
    tensors["workspace"] = std::make_shared<AsTensor>("workspace", DeviceType::CUDA, DataType::INT8, DataMode::DENSE, Shape{0});
    OperatorProto proto;
    // the layer index travels in the op name like in a serialized model ("decoder.layer.<i>.attention", common.h:239-257)
    proto.op_type_ = "DecOptMQA";
    proto.op_name_ = layer_id >= 0 ? "decoder.layer." + std::to_string(layer_id) + ".attention" : "attention_without_layer";
    proto.inputs_.push_back({"qkv"}); proto.outputs_.push_back({"attn_out"});
    auto op = OpFactory::getInstance().GetOperator({"DecOptMQA", DeviceType::CUDA})();
    AsStatus st = op->InitV2(proto, ctx, weights, weights_buffer, &tensors, &rt);
    if (st != AsStatus::ALLSPARK_SUCCESS) return (int)st;
    st = op->CallReshape(&rt);
    if (st != AsStatus::ALLSPARK_SUCCESS) return (int)st;
    for (int t = 0; t < steps; ++t) {
      tensors["qkv"]->CopyDataFrom((const char*)qkv_all + (size_t)t * batch * W * 2, (size_t)batch * W * 2, DeviceType::CPU);
      st = op->CallAlloc(&rt);
      if (st != AsStatus::ALLSPARK_SUCCESS) return (int)st;
      st = op->CallForward(&rt);
      if (st != AsStatus::ALLSPARK_SUCCESS) return (int)st;
      ctx.Synchronize();
      tensors["attn_out"]->CopyDataTo((char*)out_all + (size_t)t * batch * OW * 2, (size_t)batch * OW * 2, DeviceType::CPU);
      for (int b = 0; b < batch; ++b) rt.GetGenCtx(b)->step += 1;
    }
    return cudaGetLastError() == cudaSuccess ? 0 : -3;
  } catch (const std::exception& e) {
    AS_LOG_ERROR("as_test_span_attn: %s", e.what());
    return -1;
  }
}

// QKLayerNormNoBeta on a rank of an nranks-way tensor-parallel context: attributes num_heads / multi_query_group_num are the
// whole model's, the op divides them.  x_host / out_host [batch][(nH/nranks + 2 nG') * head_dim] in the test dtype, nG' as
// the op derives it; q_gamma_host / k_gamma_host [head_dim].
int as_test_qk_layernorm(int nranks, int batch, int num_heads, int groups, int head_dim, float eps, const void* x_host,
                         const void* q_gamma_host, const void* k_gamma_host, void* out_host) {
  try {
    CUDAContext ctx;
    ctx.SetDtype(g_test_ft);
    ctx.SetRank(0, nranks);
    const int nH = num_heads / nranks, nG = groups != 1 ? groups / nranks : 1;
    const int64_t W = (int64_t)(nH + 2 * nG) * head_dim;
    TensorMap tensors, weights, weights_buffer;
    auto add = [&](TensorMap& m, const std::string& name, Shape s, const void* src) {
      auto t = std::make_shared<AsTensor>(name, DeviceType::CUDA, g_test_ft, DataMode::DENSE, s);
      t->CopyDataFrom(src, t->GetSizeInByte(), DeviceType::CPU);
      m[name] = t;
    };
    add(tensors, "qkv", Shape{batch, 1, W}, x_host);
    add(weights, "q_norm.weight", Shape{head_dim}, q_gamma_host);
    add(weights, "k_norm.weight", Shape{head_dim}, k_gamma_host);
    OperatorProto proto;
    proto.op_type_ = "QKLayerNormNoBeta"; proto.op_name_ = "decoder.layer.0.attention.qk_norm";
    proto.inputs_.push_back({"qkv"}); proto.outputs_.push_back({"qkv_normed"});
    proto.weights_.push_back({"q_norm.weight"}); proto.weights_.push_back({"k_norm.weight"});
    proto.SetAttr<float>("eps", eps);
    proto.SetAttr<int>("num_heads", num_heads);
    proto.SetAttr<int>("multi_query_group_num", groups);
    auto op = OpFactory::getInstance().GetOperator({"QKLayerNormNoBeta", DeviceType::CUDA})();
    AsStatus st = op->InitV2(proto, ctx, weights, weights_buffer, &tensors, nullptr);
    if (st != AsStatus::ALLSPARK_SUCCESS) return (int)st;
    st = op->Reshape();
    if (st != AsStatus::ALLSPARK_SUCCESS) return (int)st;
    st = op->Forward();
    if (st != AsStatus::ALLSPARK_SUCCESS) return (int)st;
    ctx.Synchronize();
    auto out = tensors["qkv_normed"];
    if (out->GetShape().Count() != (int64_t)batch * W) return -2;
    out->CopyDataTo(out_host, out->GetSizeInByte(), DeviceType::CPU);
    return cudaGetLastError() == cudaSuccess ? 0 : -3;
  } catch (const std::exception& e) {
    AS_LOG_ERROR("as_test_qk_layernorm: %s", e.what());
    return -1;
  }
}

// RotaryMulQuery with the attributes of the reference's GLM converter (head counts of the whole model, one rank) on x_host
// [batch][(num_heads + 2 groups) * head_dim] in the test dtype at positions pos_host[b] (gen_ctx->step); out_host receives the
// rotated rows.  Returns the AsStatus of the first step that fails (Init refuses unsupported rotary / invfreq types).
int as_test_rotary_mulquery(int batch, int num_heads, int groups, int hidden_size, int rotary_type, int invfreq_type,
                            float rope_ratio, float rotary_base, const int* pos_host, const void* x_host, void* out_host) {
  try {
    CUDAContext ctx;
    ctx.SetDtype(g_test_ft);
    const int head_dim = hidden_size / num_heads;
    const int64_t W = (int64_t)(num_heads + 2 * groups) * head_dim;
    TensorMap tensors, weights, weights_buffer;
    auto t = std::make_shared<AsTensor>("qkv", DeviceType::CUDA, g_test_ft, DataMode::DENSE, Shape{batch, 1, W});
    t->CopyDataFrom(x_host, t->GetSizeInByte(), DeviceType::CPU);
    tensors["qkv"] = t;
    RuntimeContext rt(false);
    for (int b = 0; b < batch; ++b) {
      auto g = std::make_unique<GenerateContext>();
      g->step = pos_host[b];
      rt.PushBackGenCtx(std::move(g));
    }
    OperatorProto proto;
    proto.op_type_ = "RotaryMulQuery"; proto.op_name_ = "decoder.layer.0.rotary";
    proto.inputs_.push_back({"qkv"}); proto.outputs_.push_back({"qkv_rotary"});
    proto.SetAttr<int>("num_heads", num_heads);
    proto.SetAttr<int>("multi_query_group_num", groups);
    proto.SetAttr<int>("hidden_size", hidden_size);
    proto.SetAttr<int>("rotary_type", rotary_type);
    proto.SetAttr<int>("invfreq_type", invfreq_type);
    proto.SetAttr<float>("rope_ratio", rope_ratio);
    proto.SetAttr<float>("rotary_base", rotary_base);
    auto op = OpFactory::getInstance().GetOperator({"RotaryMulQuery", DeviceType::CUDA})();
    AsStatus st = op->InitV2(proto, ctx, weights, weights_buffer, &tensors, &rt);
    if (st != AsStatus::ALLSPARK_SUCCESS) return (int)st;
    st = op->CallReshape(&rt);
    if (st != AsStatus::ALLSPARK_SUCCESS) return (int)st;
    st = op->CallForward(&rt);
    if (st != AsStatus::ALLSPARK_SUCCESS) return (int)st;
    ctx.Synchronize();
    auto out = tensors["qkv_rotary"];
    if (out->GetShape().Count() != (int64_t)batch * W) return -2;
    out->CopyDataTo(out_host, out->GetSizeInByte(), DeviceType::CPU);
    return cudaGetLastError() == cudaSuccess ? 0 : -3;
  } catch (const std::exception& e) {
    AS_LOG_ERROR("as_test_rotary_mulquery: %s", e.what());
    return -1;
  }
}

}  // extern "C"
