"""GPU: DecodeStack.launches_per_step is the number of kernels its step puts on the GPU.  For each configuration the step is
recorded once more into a CUDA graph that is kept and not replayed, and the graph's kernel nodes are counted through the
driver API (cuGraphGetNodes, cuGraphNodeGetType); memcpy and memset nodes are not launches.  The configurations cover
every feature of the step, the three norm placements, the GEMM row chunks (64 rows per wgmma launch, 16 per mma.sync
launch for sub-channel int8 weights), fp16, head 64, a batch re-viewed by set_batch, and stacks whose features the tools
switch off between captures."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

CU_GRAPH_NODE_TYPE_KERNEL = 0

# (id, model, construction batch, batch the steps run with (set_batch), DecodeStack keywords); TINY: 2 layers, head 128
CONFIGS = [
    *[("b%d" % B, "TINY", B, B, {}) for B in (1, 2, 5, 17, 64)],
    ("b64-view8", "TINY", 64, 8, {}),
    ("q4-b20", "TINY", 20, 20, dict(q_len=4)),  # R = 80 rows: two launches per GEMM
    ("int8-g128-b2", "TINY", 2, 2, dict(wbits=8, group=128)),
    ("int8-g128-b17", "TINY", 17, 17, dict(wbits=8, group=128)),  # 16-row chunks: two launches per projection
    ("int8-g128-b64", "TINY", 64, 64, dict(wbits=8, group=128)),
    ("int8-b17", "TINY", 17, 17, dict(wbits=8)),
    ("dense-g128-b17", "TINY", 17, 17, dict(wbits=16, group=128)),  # dense weights ignore the group: 64-row chunks
    ("int4-g72-b5", "TINY", 5, 5, dict(group=72, fuse_swiglu=False)),
    ("int4-g72-b17", "TINY", 17, 17, dict(group=72, fuse_swiglu=False)),
    ("unfused-b1", "TINY", 1, 1, dict(fuse_swiglu=False)),
    ("unfused-b17", "TINY", 17, 17, dict(fuse_swiglu=False)),
    ("fp16-b2", "TINY", 2, 2, dict(dtype=torch.float16)),
    ("fp16-b17", "TINY", 17, 17, dict(dtype=torch.float16)),
    ("head64-b3", "QWEN2_05B", 3, 3, dict(layers=1)),
    ("head64-b17", "QWEN2_05B", 17, 17, dict(layers=1)),
    ("logprobs-b1", "TINY", 1, 1, dict(logprobs=5)),
    ("logprobs-b17", "TINY", 17, 17, dict(logprobs=10)),
    ("sample-b1", "TINY", 1, 1, dict(sample=True)),
    ("sample-b17", "TINY", 17, 17, dict(sample=True)),
    ("sample-logprobs-b5", "TINY", 5, 5, dict(sample=True, logprobs=3)),
    ("penalties-b5", "TINY", 5, 5, dict(penalties=True)),
    ("penalties-sample-b17", "TINY", 17, 17, dict(penalties=True, sample=True, logprobs=2)),
    ("chain-q4-b3", "TINY", 3, 3, dict(q_len=4)),
    ("logprobs-q4-b3", "TINY", 3, 3, dict(q_len=4, logprobs=4)),
    ("tree-q4-b3", "TINY", 3, 3, dict(q_len=4, tree=True)),
    ("tree-q8-b8", "TINY", 8, 8, dict(q_len=8, tree=True)),
    ("sv-chain-q4-b3", "TINY", 3, 3, dict(q_len=4, sampled_verify=True)),
    ("sv-tree-q8-b4", "TINY", 4, 4, dict(q_len=8, tree=True, sampled_verify=True)),
    ("sv-logprobs-q4-b5", "TINY", 5, 5, dict(q_len=4, sampled_verify=True, logprobs=3)),
    ("sv-tree-logprobs-q4-b3", "TINY", 3, 3, dict(q_len=4, tree=True, sampled_verify=True, logprobs=3)),
    ("ngram-chain-q4-b4", "TINY", 4, 4, dict(q_len=4, ngram=(1, 3, 1))),
    ("ngram-tree-q8-b4", "TINY", 4, 4, dict(q_len=8, tree=True, ngram=(1, 3, 3))),
    ("ngram-sv-tree-q8-b4", "TINY", 4, 4, dict(q_len=8, tree=True, sampled_verify=True, ngram=(2, 4, 2))),
]


# The tools capture one stack in two forms by switching a feature off between captures (tools/spec_bench.py,
# penalty_bench.py, sample_bench.py, logprobs_bench.py): (id, model, batch, batch the steps run with, DecodeStack keywords,
# flags set before the capture)
SWITCHED = [
    ("tree-off-q4-b3", "TINY", 3, 3, dict(q_len=4, tree=True), dict(tree=False)),
    ("sv-tree-off-q8-b4", "TINY", 4, 4, dict(q_len=8, tree=True, sampled_verify=True), dict(tree=False)),
    ("sv-off-tree-q8-b4", "TINY", 4, 4, dict(q_len=8, tree=True, sampled_verify=True), dict(sv=False)),
    ("sv-off-tree-off-q4-b3", "TINY", 3, 3, dict(q_len=4, tree=True, sampled_verify=True), dict(sv=False, tree=False)),
    ("ngram-tree-off-q8-b4", "TINY", 4, 4, dict(q_len=8, tree=True, ngram=(1, 4, 3)), dict(tree=False, ngram=(1, 4, 1))),
    ("ngram-off-tree-q8-b4", "TINY", 4, 4, dict(q_len=8, tree=True, ngram=(1, 4, 3)), dict(ngram=None)),
    ("ngram-off-tree-off-q4-b4", "TINY", 4, 4, dict(q_len=4, tree=True, ngram=(1, 4, 1)), dict(tree=False, ngram=None)),
    ("penalties-off-b5", "TINY", 5, 5, dict(penalties=True), dict(pen=False)),
    ("sample-off-b17", "TINY", 17, 17, dict(sample=True), dict(sample=False)),
    ("logprobs-off-b5", "TINY", 5, 5, dict(logprobs=4), dict(logprobs=0)),
]


def make_stack(model_name, B, b, kw, flags=None):
    from b200spark import model
    st = model.DecodeStack(getattr(model, model_name), B, 160, span=16, seed=5, **kw)
    st.set_batch(b)
    for k, v in (flags or {}).items():
        setattr(st, k, v)
    return st


def graph_kernels(graph):
    """The kernel nodes of a graph captured with keep_graph=True, in the driver's order."""
    cu = ctypes.CDLL("libcuda.so.1")
    g = ctypes.c_void_p(graph.raw_cuda_graph())
    n = ctypes.c_size_t(0)
    assert cu.cuGraphGetNodes(g, None, ctypes.byref(n)) == 0
    nodes = (ctypes.c_void_p * n.value)()
    assert cu.cuGraphGetNodes(g, nodes, ctypes.byref(n)) == 0
    kind = ctypes.c_int()
    kernels = []
    for node in nodes[:n.value]:
        assert cu.cuGraphNodeGetType(ctypes.c_void_p(node), ctypes.byref(kind)) == 0
        if kind.value == CU_GRAPH_NODE_TYPE_KERNEL:
            kernels.append(node)
    return kernels


def recorded_step(st):
    """st.capture(), then the step recorded once more into a graph that is kept for inspection and never replayed"""
    st.capture()
    g = torch.cuda.CUDAGraph(keep_graph=True)
    with torch.cuda.graph(g):
        st._step_ops()
    torch.cuda.synchronize()
    return g


@pytest.mark.parametrize("name,model_name,B,b,kw", CONFIGS, ids=[c[0] for c in CONFIGS])
def test_launch_count_equals_graph_kernels(name, model_name, B, b, kw):
    st = make_stack(model_name, B, b, kw)
    g = recorded_step(st)
    assert len(graph_kernels(g)) == st.launches_per_step > 0, name


@pytest.mark.parametrize("name,model_name,B,b,kw,flags", SWITCHED, ids=[c[0] for c in SWITCHED])
def test_launch_count_with_a_feature_switched_off(name, model_name, B, b, kw, flags):
    st = make_stack(model_name, B, b, kw, flags)
    g = recorded_step(st)
    assert len(graph_kernels(g)) == st.launches_per_step > 0, name
