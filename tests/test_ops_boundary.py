"""The ops boundary, without a GPU: every status-returning entry point is called through ``ops._call``, every pointer comes from
``ops._arg``, and every public wrapper that reaches the library refuses CPU tensors before it calls a compute entry point."""
import ast
from pathlib import Path

import pytest
import torch

from dance_b200 import ops
from dance_b200._lib import B2Error

PKG = Path(ops.__file__).resolve().parent
SOURCES = {name: ast.parse((PKG / name).read_text()) for name in ("ops.py", "parallel.py")}

# entry points that return a value rather than a status: called directly
QUERIES = {"b2_gae_sym_super_blocks", "b2_get_path", "b2_launch_count", "b2_version", "b2_last_error", "b2_comm_available"}


def _is_query(name: str) -> bool:
    return name in QUERIES or name.endswith("_workspace_bytes")


def _functions(tree):
    """{name: node} of the module-level functions and of the methods (as Class.method)."""
    out = {}
    for node in tree.body:
        if isinstance(node, (ast.FunctionDef, ast.ClassDef)):
            out[node.name] = node
            if isinstance(node, ast.ClassDef):
                out.update({f"{node.name}.{m.name}": m for m in node.body if isinstance(m, ast.FunctionDef)})
    return out


def _called_names(node):
    return {n.func.id if isinstance(n.func, ast.Name) else n.func.attr for n in ast.walk(node) if isinstance(n, ast.Call)
            and isinstance(n.func, (ast.Name, ast.Attribute))}


@pytest.mark.parametrize("module", sorted(SOURCES))
def test_only_queries_are_called_directly(module):
    direct = sorted({n.attr for n in ast.walk(SOURCES[module]) if isinstance(n, ast.Attribute) and n.attr.startswith("b2_")
                     and not _is_query(n.attr)})
    assert direct == [], f"{module} calls {direct} outside ops._call"
    assert "check" not in _called_names(SOURCES[module])


@pytest.mark.parametrize("module", sorted(SOURCES))
def test_pointers_come_from_the_accessor(module):
    users = sorted({name for name, fn in _functions(SOURCES[module]).items() if isinstance(fn, ast.FunctionDef) and any(
        isinstance(n, ast.Attribute) and n.attr == "data_ptr" for n in ast.walk(fn))})
    assert users == (["_arg"] if module == "ops.py" else [])


def _reaching_call():
    """Public module-level functions of ops that reach ``_call``, directly or through other functions of the module."""
    fns = {k: v for k, v in _functions(SOURCES["ops.py"]).items() if isinstance(v, ast.FunctionDef) and "." not in k}
    calls = {k: _called_names(v) for k, v in fns.items()}
    reach = {"_call"}
    while True:
        more = {k for k, c in calls.items() if c & reach} - reach
        if not more:
            return sorted(k for k in reach if not k.startswith("_"))
        reach |= more


class Recorder:
    """Stands in for the ctypes library: answers the queries and records every other call."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        if name == "b2_last_error":
            return lambda: b"recorded"
        if _is_query(name):
            return lambda *a: 1 << 10 if name.endswith("_bytes") else 1
        return lambda *a: self.calls.append(name) or 0


def _fake_csr(n=6, nnz=10, vals=True):
    """A CSR whose tensors live on the CPU (CSR() itself refuses them): what a wrapper would see if that check were missing."""
    A = ops.CSR.__new__(ops.CSR)
    A.rowptr = torch.arange(0, n + 1, dtype=torch.int32).clamp(max=nnz)
    A.colidx = torch.zeros(nnz, dtype=torch.int32)
    A.vals = torch.ones(nnz) if vals else None
    A.shape, A.ptrs, A._t = (n, n), (1, 1, 1 if vals else None), None
    return A


f32 = lambda *s: torch.zeros(*s, dtype=torch.float32)
i32 = lambda *s: torch.zeros(*s, dtype=torch.int32)

# one call per public wrapper that reaches the library, with CPU tensors throughout
CASES = {
    "to_x16": lambda: ops.to_x16(f32(4, 8)),
    "spmm": lambda: ops.spmm(_fake_csr(), f32(6, 8)),
    "csr_transpose": lambda: ops.csr_transpose(_fake_csr()),
    "gemm": lambda: ops.gemm(f32(4, 4), f32(4, 4)),
    "colsum": lambda: ops.colsum(f32(4, 4)),
    "mse_sum_loss_grad": lambda: ops.mse_sum_loss_grad(f32(4, 4), f32(4, 4)),
    "gae_loss_grad": lambda: ops.gae_loss_grad(f32(6, 8), _fake_csr(vals=False), 1.0, 1.0),
    "gae_loss_grad_sym": lambda: ops.gae_loss_grad_sym(f32(6, 8), _fake_csr(vals=False), 1.0, 1.0, 0, 1),
    "adam_step": lambda: ops.adam_step(f32(4), f32(4), f32(4), f32(4), 1),
    "reparam_fwd": lambda: ops.reparam_fwd(f32(4, 8), f32(4, 8), f32(4, 8)),
    "reparam_bwd": lambda: ops.reparam_bwd(f32(4, 8), f32(4, 8), f32(4, 8), f32(4, 8), f32(4, 8)),
    "knn": lambda: ops.knn(f32(8, 4), 2),
    "pairwise_l2_dense": lambda: ops.pairwise_l2_dense(f32(8, 4)),
    "knn_graph_build": lambda: ops.knn_graph_build(i32(8, 2)),
    "knn_graph_weighted_build": lambda: ops.knn_graph_weighted_build(i32(8, 2), torch.zeros(8, 2, dtype=torch.float64)),
    "normalize_total_log1p_": lambda: ops.normalize_total_log1p_(f32(4, 4)),
    "dropout": lambda: ops.dropout(f32(4, 4), 0.5, 0, 0),
    "gat_scores": lambda: ops.gat_scores(f32(6, 8), f32(8), f32(8), 2),
    "gat_aggregate_fwd": lambda: ops.gat_aggregate_fwd(_fake_csr(vals=False), f32(6, 8), f32(6, 2), f32(6, 2), 2),
    "gat_aggregate_bwd": lambda: ops.gat_aggregate_bwd(_fake_csr(vals=False), _fake_csr(vals=False), i32(10), f32(6, 8), f32(8), f32(8),
                                                       f32(6, 2), f32(6, 2), f32(10, 2), f32(6, 8), 2),
    "gat_combine_fwd": lambda: ops.gat_combine_fwd(f32(6, 8), None, None, 2, True),
    "gat_combine_bwd": lambda: ops.gat_combine_bwd(f32(6, 8), f32(6, 8), 2, 4, True),
    "cellgene_graph": lambda: ops.cellgene_graph(f32(4, 4)),
    "sage_edge_values": lambda: ops.sage_edge_values(_fake_csr(), f32(10), f32(6), 4),
    "softmax_ce_sum": lambda: ops.softmax_ce_sum(f32(4, 3), torch.zeros(4, dtype=torch.int64)),
    "sym_eig": lambda: ops.sym_eig(f32(4, 4)),
    "pca": lambda: ops.pca(f32(8, 4), 2),
    "dec_q": lambda: ops.dec_q(f32(6, 4), f32(3, 4)),
    "dec_target": lambda: ops.dec_target(f32(6, 3)),
    "dec_kl_grad": lambda: ops.dec_kl_grad(f32(6, 4), f32(3, 4), f32(6, 3)),
    "sgd_momentum_step": lambda: ops.sgd_momentum_step(f32(4), f32(4), f32(4), 1, 0.1),
    "exp_adj": lambda: ops.exp_adj(f32(4, 4), 1.0),
    "clip_grad_norm_": lambda: ops.clip_grad_norm_(f32(4), 1.0),
    "radius_graph": lambda: ops.radius_graph(torch.zeros(4, 2, dtype=torch.float64), 1.0),
    "matrix_normalize": lambda: ops.matrix_normalize(f32(4, 4)),
    "pearson_corr": lambda: ops.pearson_corr(f32(4, 4)),
    "threshold_graph": lambda: ops.threshold_graph(f32(4, 4), 0.5),
    "umap_connectivities": lambda: ops.umap_connectivities(i32(8, 3), f32(8, 3)),
    "batchnorm_fwd": lambda: ops.batchnorm_fwd(f32(6, 4), f32(4), f32(4), f32(4), f32(4), True),
    "batchnorm_bwd": lambda: ops.batchnorm_bwd(f32(6, 4), None, f32(6, 4), f32(4), f32(4), f32(4)),
    "zinb_loss_grad": lambda: ops.zinb_loss_grad(f32(4, 4), f32(4, 4), f32(4, 4), f32(4, 4), f32(4)),
    "adj_sample": lambda: ops.adj_sample(f32(4, 4), f32(4, 4), f32(4, 4)),
    "adj_loss_grad": lambda: ops.adj_loss_grad(f32(4, 4), f32(4, 4), f32(4, 4), f32(4, 4), f32(4)),
    "adj_reparam_bwd": lambda: ops.adj_reparam_bwd(f32(4, 4), f32(4, 4), f32(4, 4), f32(4, 4), 1.0),
    "kmeans": lambda: ops.kmeans(f32(8, 4), f32(2, 4)),
    "graph_regu_weights": lambda: ops.graph_regu_weights(_fake_csr(), i32(6), n_clusters=2),
    "graph_regu_weights_weighted": lambda: ops.graph_regu_weights_weighted(i32(7), i32(10), torch.zeros(10, dtype=torch.float64), i32(6),
                                                                           n_clusters=2),
    "celltype_loss_grad": lambda: ops.celltype_loss_grad(f32(4, 4), f32(4, 4), f32(4, 4), f32(4)),
    "l1_grad_add": lambda: ops.l1_grad_add(f32(4), f32(4)),
    "gene_stats": lambda: ops.gene_stats(f32(4, 4)),
    "cell_stats": lambda: ops.cell_stats(f32(4, 4)),
    "subset": lambda: ops.subset(f32(4, 4)),
    "cellwise_mask": lambda: ops.cellwise_mask(f32(4, 4)),
    "locality_order": lambda: ops.locality_order(f32(8, 4)),
    "quantiles": lambda: ops.quantiles(f32(4, 4), 0.5),
    "col_minmax": lambda: ops.col_minmax(f32(4, 4)),
    "concat_normalized": lambda: ops.concat_normalized(f32(4, 4), f32(4, 4)),
    "act": lambda: ops.act(f32(4, 4), "gelu"),
    "act_bwd": lambda: ops.act_bwd(f32(4, 4), "relu", y=f32(4, 4)),
    "graphsc_block_degrees": lambda: ops.graphsc_block_degrees(_fake_csr(), i32(3)),
    "graphsc_block_aggregate": lambda: ops.graphsc_block_aggregate(_fake_csr(), i32(3), i32(6), f32(6, 4)),
    "graphsc_batch_decoder": lambda: ops.graphsc_batch_decoder(f32(4, 4)),
    "graphsc_scatter_rows": lambda: ops.graphsc_scatter_rows(f32(4, 4), i32(4), f32(8, 4)),
}
# wrappers that hand the library no device tensor
NO_DEVICE_TENSORS = {"set_path", "set_tuning", "device_info", "louvain_host"}


def test_case_table_names_every_wrapper():
    reach = set(_reaching_call())
    assert reach - NO_DEVICE_TENSORS == set(CASES), "a public ops function that reaches the library has no CPU-tensor case"
    assert len(reach) > 60


@pytest.fixture
def recorder(monkeypatch):
    rec = Recorder()
    monkeypatch.setattr(ops, "_raw_lib", lambda: rec)
    return rec


@pytest.mark.parametrize("name", sorted(CASES))
def test_ops_refuse_cpu_tensors(recorder, name):
    with pytest.raises(B2Error, match="expected a CUDA tensor"):
        CASES[name]()
    assert recorder.calls == []


def test_csr_refuses_cpu_tensors():
    with pytest.raises(B2Error, match="expected a CUDA tensor"):
        ops.CSR(torch.tensor([0, 1], dtype=torch.int32), torch.tensor([0], dtype=torch.int32), None, (1, 1))


def test_call_raises_with_the_entry_point_and_the_library_message(monkeypatch):
    rec = Recorder()
    monkeypatch.setattr(ops, "_raw_lib", lambda: rec)
    monkeypatch.setattr(Recorder, "__getattr__", lambda self, name: (lambda *a: b"bad arguments") if name == "b2_last_error"
                        else (lambda *a: -1))
    with pytest.raises(B2Error, match=r"^b2_set_path failed with status -1: bad arguments$"):
        ops.set_path("gae", "auto")
