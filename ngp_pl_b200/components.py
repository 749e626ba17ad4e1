"""Connected components of the occupancy grid on the device: remove floaters from a trained model's density_bitfield.

    occupancy_components(model) -> labels, sizes      (cascades * G^3,) int32 each, on the model's device
    remove_floaters(model, keep_largest=None, min_cells=None, return_stats=False)

The graph (include/ngp_b200.h, "Connected components"): the occupied cells of each cascade's shell -- every cell of
cascade 0, and the cells of cascade c >= 1 not wholly inside cascade c - 1's box -- joined by 26-adjacency inside a
cascade and by closed-box contact with the next finer cascade. A cell's label is the smallest cell index of its
component (cell c G^3 + morton(x, y, z), the bitfield's order), -1 for cells that are not nodes; sizes holds each
component's cell count at its label. Every consumer of the bitfield (render, show_gui, export_points,
extract_mesh_sparse, metrics.evaluate) sees the cleaned grid without any change of its own.

Kernels: `ngp_grid_components`, `ngp_components_select`, `ngp_grid_components_clean` (csrc/components.cu). Model and
bitfield must live on a CUDA device, otherwise RuntimeError; there is no CPU path.
"""
import ctypes as C

import torch

from . import _lib

INT64_MAX = (1 << 63) - 1


def _st(dev):
    return torch.cuda.current_stream(dev).cuda_stream


def criterion(v, name, fn):
    """None, or v as a positive int (RuntimeError otherwise)"""
    if v is None:
        return None
    if isinstance(v, (bool, float)) or not hasattr(v, "__index__") or int(v) < 1:
        raise RuntimeError("ngp_pl_b200.%s: %s must be a positive integer, got %r" % (fn, name, v))
    return int(v)


def select_components(labels, sizes, keep_largest, min_size, fn):
    """keep (n,) uint8 on the labels' device -- 1 at the label of every component that is among the keep_largest
    largest (ties to the smaller label) and has at least min_size nodes -- and {'components', 'kept'}. None leaves a
    criterion out (the callers have checked them with criterion() and require at least one)."""
    n = labels.numel()
    dev = labels.device
    L = _lib.lib()
    with torch.cuda.device(dev):
        ws_bytes = L.ngp_components_select_workspace(n)
        if ws_bytes == 0:
            raise RuntimeError("ngp_pl_b200.%s: %d nodes: must be below 2^31" % (fn, n))
        ws = torch.empty(ws_bytes, device=dev, dtype=torch.uint8)
        keep = torch.empty(n, device=dev, dtype=torch.uint8)
        cnt = (C.c_int64 * 2)()
        _lib.check(L.ngp_components_select(labels.data_ptr(), sizes.data_ptr(), n,
                                           INT64_MAX if keep_largest is None else keep_largest,
                                           0 if min_size is None else min_size, keep.data_ptr(), cnt, ws.data_ptr(),
                                           ws_bytes, _st(dev)), "ngp_components_select")
    return keep, {"components": int(cnt[0]), "kept": int(cnt[1])}


def _grid(model, fn):
    bits = model.density_bitfield
    if not bits.is_cuda:
        raise RuntimeError("ngp_pl_b200.components.%s needs the model on a CUDA device (got %s); there is no CPU path"
                           % (fn, bits.device))
    G, C_ = int(model.grid_size), int(model.cascades)
    if bits.dtype != torch.uint8 or bits.numel() * 8 != C_ * G ** 3 or not bits.is_contiguous():
        raise RuntimeError("ngp_pl_b200.components.%s: density_bitfield must be %d contiguous bytes (%d cascades of "
                           "%d^3 cells), got %s %s" % (fn, C_ * G ** 3 // 8, C_, G, tuple(bits.shape), bits.dtype))
    return bits, C_, G, float(model.scale)


@torch.no_grad()
def occupancy_components(model):
    """(labels, sizes) of model.density_bitfield's occupancy graph, each (cascades * G^3,) int32 on its device:
    labels[i] = the smallest cell index of cell i's component (-1 for an empty or an inner cell), sizes[l] = the number
    of cells of the component labelled l (0 at every index that is not a label). Deterministic: two calls are bitwise
    equal."""
    bits, C_, G, scale = _grid(model, "occupancy_components")
    n = C_ * G ** 3
    dev = bits.device
    labels = torch.empty(n, device=dev, dtype=torch.int32)
    sizes = torch.empty(n, device=dev, dtype=torch.int32)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().ngp_grid_components(bits.data_ptr(), C_, G, scale, labels.data_ptr(), sizes.data_ptr(),
                                                  _st(dev)), "ngp_grid_components")
    return labels, sizes


@torch.no_grad()
def remove_floaters(model, keep_largest=None, min_cells=None, return_stats=False):
    """Clear the occupancy of every component of the occupancy graph that is not among the keep_largest largest or has
    fewer than min_cells cells (at least one criterion is required; with both, a component must pass both). Inner
    cells -- cells of cascade c >= 1 inside cascade c - 1's box, which the marcher never reads where the finer cascade
    reaches -- follow the finer cascade: one is cleared when the finer cells its box meets include a cleared cell and
    none left occupied. Edits model.density_bitfield in place and, when the model has a registered density_grid, sets
    the cleared cells to -1 there, so update_density_grid never revives them. Returns the model; return_stats=True
    also returns {'components', 'kept', 'cleared_cells', 'cleared_inner'}."""
    bits, C_, G, scale = _grid(model, "remove_floaters")
    dev = bits.device
    dg = model._buffers.get("density_grid")
    if dg is not None and (not dg.is_cuda or dg.device != dev or dg.dtype != torch.float32 or dg.numel() != C_ * G ** 3
                           or not dg.is_contiguous()):
        raise RuntimeError("ngp_pl_b200.components.remove_floaters: density_grid must be a contiguous (%d, %d) float32 "
                           "tensor on %s, got %s %s on %s" % (C_, G ** 3, dev, tuple(dg.shape), dg.dtype, dg.device))
    keep_largest = criterion(keep_largest, "keep_largest", "components.remove_floaters")
    min_cells = criterion(min_cells, "min_cells", "components.remove_floaters")
    if keep_largest is None and min_cells is None:
        raise RuntimeError("ngp_pl_b200.components.remove_floaters: give keep_largest, min_cells, or both")
    labels, sizes = occupancy_components(model)
    keep, stats = select_components(labels, sizes, keep_largest, min_cells, "components.remove_floaters")
    with torch.cuda.device(dev):
        removed = torch.empty(bits.numel(), device=dev, dtype=torch.uint8)
        cleared = torch.empty(2, device=dev, dtype=torch.int64)
        _lib.check(_lib.lib().ngp_grid_components_clean(bits.data_ptr(), None if dg is None else dg.data_ptr(), C_, G,
                                                        scale, labels.data_ptr(), keep.data_ptr(), removed.data_ptr(),
                                                        cleared.data_ptr(), _st(dev)), "ngp_grid_components_clean")
    if return_stats:
        shell, inner = (int(x) for x in cleared.cpu())
        stats.update(cleared_cells=shell, cleared_inner=inner)
        return model, stats
    return model
