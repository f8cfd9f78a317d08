"""Import the UNMODIFIED reference (the `src/` directory of an enoche/MMRec checkout, named by the environment
variable MMREC_REFERENCE_SRC).

Only `tests/golden/make_golden.py` and `tools/ref_vs_port_timing.py` use this; the tests read the committed
golden files only.  Nothing is copied: the reference is put on `sys.path` and
four import-time breakages of its environment pins (torch 1.11 / numpy 1.21 /
scipy 1.7, `requirements.txt`) are shimmed, as listed in SURVEY.md Appendix A:

* `lmdb`, `matplotlib` -- imported but unused on this path
  (`src/utils/dataset.py:18`, `src/common/trainer.py:14`) -> empty stub modules;
* `scipy.sparse.dok_matrix._update` -- private API removed from scipy
  (`src/models/freedom.py:111`) -> dict update;
* `np.float` -- removed alias (`src/utils/metrics.py:51`);
* `torch_scatter.scatter_add` (`src/utils/utils.py:140`, MGCN only) -> index_add_;
* MGCN hard-codes `.cuda()` (`src/models/mgcn.py:59,69`) -> identity on a CPU box;
* LayerGCN imports `models.common.*` (`src/models/layergcn.py:12-13`) -> alias;
* MMGCN imports `torch_geometric` (`src/models/mmgcn.py:13-15`; the reference pins no version, the package is not
  installable here) -> `install_pyg_shim()`: the three things the file uses, restated from PyG's documented behaviour --
  `MessagePassing(aggr=...)` with the default flow `source_to_target` (`x_j = x[edge_index[0]]`, aggregated at
  `edge_index[1]`, 'mean' = sum / in-degree, untouched nodes 0), `nn.inits.uniform` (U(-1/sqrt(size), 1/sqrt(size))) and the
  unused `utils` names.  With it the reference's OWN model code (towers, loss, scoring: `mmgcn.py:22-188`) runs
  unmodified; what stays restated is that one primitive.
"""
import os
import sys
import types

import numpy as np
import scipy.sparse as sp
import torch

REF_SRC = os.environ.get("MMREC_REFERENCE_SRC", "")             # src/ of an enoche/MMRec checkout


def install():
    if not os.path.isdir(REF_SRC):
        raise RuntimeError("set MMREC_REFERENCE_SRC to the src/ directory of an unmodified enoche/MMRec checkout")
    for name in ("lmdb", "matplotlib", "matplotlib.pyplot"):
        sys.modules.setdefault(name, types.ModuleType(name))
    ts = types.ModuleType("torch_scatter")
    ts.scatter_add = lambda src, index, dim=0, dim_size=None: torch.zeros(
        dim_size, dtype=src.dtype, device=src.device).index_add_(0, index, src)
    sys.modules.setdefault("torch_scatter", ts)
    if not hasattr(sp.dok_matrix, "_update"):
        sp.dok_matrix._update = lambda self, d: self._dict.update({k: np.float32(v) for k, v in d.items()})
    if not hasattr(np, "float"):
        np.float = float
    if not torch.cuda.is_available():
        torch.Tensor.cuda = lambda self, *a, **k: self
    if REF_SRC not in sys.path:
        sys.path.insert(0, REF_SRC)
    import common
    import common.abstract_recommender
    import common.loss
    for m in ("", ".abstract_recommender", ".loss"):
        sys.modules["models.common" + m] = sys.modules["common" + m]


def install_pyg_shim():
    """`torch_geometric` as far as `src/models/mmgcn.py` uses it (see the module docstring)."""
    if "torch_geometric" in sys.modules:
        return

    class MessagePassing(torch.nn.Module):
        def __init__(self, aggr="add", flow="source_to_target", **kwargs):
            super().__init__()
            self.aggr, self.flow = aggr, flow

        def propagate(self, edge_index, size=None, **kwargs):
            src, dst = (edge_index[0], edge_index[1]) if self.flow == "source_to_target" else (edge_index[1], edge_index[0])
            x = kwargs["x"]
            n_out = x.size(0) if size is None else size[1]
            msg = self.message(x_j=x.index_select(0, src), edge_index=edge_index, size=size)
            out = torch.zeros(n_out, msg.size(1), dtype=msg.dtype, device=msg.device).index_add_(0, dst, msg)
            if self.aggr == "mean":
                cnt = torch.zeros(n_out, dtype=msg.dtype, device=msg.device).index_add_(0, dst, torch.ones_like(dst, dtype=msg.dtype))
                out = out / cnt.clamp(min=1).unsqueeze(1)
            elif self.aggr != "add":
                raise NotImplementedError(self.aggr)
            return self.update(out)

        def message(self, x_j, **kwargs):
            return x_j

        def update(self, aggr_out):
            return aggr_out

    def uniform(size, tensor):
        if tensor is not None:
            bound = 1.0 / (size ** 0.5)
            tensor.data.uniform_(-bound, bound)

    def degree(index, num_nodes=None, dtype=None):
        n = int(index.max()) + 1 if num_nodes is None else num_nodes
        return torch.zeros(n, dtype=dtype or torch.float32).index_add_(0, index, torch.ones_like(index, dtype=dtype or torch.float32))

    pyg = types.ModuleType("torch_geometric")
    nn_m, conv_m, inits_m, utils_m = (types.ModuleType("torch_geometric." + n) for n in ("nn", "nn.conv", "nn.inits", "utils"))
    conv_m.MessagePassing = MessagePassing
    inits_m.uniform = uniform
    utils_m.degree = degree
    utils_m.remove_self_loops = lambda edge_index, edge_attr=None: (edge_index[:, edge_index[0] != edge_index[1]], edge_attr)
    utils_m.add_self_loops = lambda edge_index, num_nodes=None: (torch.cat([edge_index, torch.arange(num_nodes).repeat(2, 1)], 1), None)
    nn_m.conv, nn_m.inits, pyg.nn, pyg.utils = conv_m, inits_m, nn_m, utils_m
    for name, m in (("torch_geometric", pyg), ("torch_geometric.nn", nn_m), ("torch_geometric.nn.conv", conv_m),
                    ("torch_geometric.nn.inits", inits_m), ("torch_geometric.utils", utils_m)):
        sys.modules[name] = m


def run_dir(tmp: str) -> str:
    """`Config` resolves `./configs` against CWD (`src/utils/configurator.py:72-73`) and the data
    path is `../data/` (`src/configs/overall.yaml:7`): build `<tmp>/run/configs -> reference` and
    return `<tmp>/data`, leaving CWD in `<tmp>/run`."""
    run = os.path.join(tmp, "run")
    os.makedirs(run, exist_ok=True)
    link = os.path.join(run, "configs")
    if not os.path.exists(link):
        os.symlink(os.path.join(REF_SRC, "configs"), link)
    os.makedirs(os.path.join(tmp, "data"), exist_ok=True)
    os.chdir(run)
    return os.path.join(tmp, "data")
