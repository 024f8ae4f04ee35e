"""Named N-D device mesh of global ranks (row-major), without torch DeviceMesh internals.

Mirror of what the lowering needs from easydist/torch/device_mesh.py: `size(dim)`,
`get_coordinate()`, the flat rank list of the sub-mesh along one dim through this rank's
coordinate (sharding.py:725-730), and the 'spmd' alias binding of dims whose name contains
"spmd" (device_mesh.py:115-121).  Unlike NDDeviceMesh it accepts size-1 dims, which is how the
"1 x H100" configuration runs through the same compiled path (the reference does not compile at
world size 1: api.py:117-118, device_mesh.py:39-41).
"""
import numpy as np


class DeviceMesh:
    def __init__(self, mesh, dim_names=None, rank=None):
        self.mesh = np.asarray(mesh, dtype=np.int64)
        if self.mesh.ndim == 0:
            self.mesh = self.mesh.reshape(1)
        self.dim_names = tuple(dim_names) if dim_names else tuple(
            f"spmd{i}" for i in range(self.mesh.ndim))
        assert len(self.dim_names) == self.mesh.ndim
        if rank is None:
            import os
            rank = int(os.environ.get("RANK", "0"))
        self.rank = int(rank)
        where = np.argwhere(self.mesh == self.rank)
        if len(where) != 1:
            raise ValueError(f"rank {self.rank} appears {len(where)} times in mesh {self.mesh}")
        self._coord = tuple(int(c) for c in where[0])

    @property
    def ndim(self):
        return self.mesh.ndim

    @property
    def shape(self):
        return tuple(self.mesh.shape)

    def size(self, mesh_dim=None):
        return int(self.mesh.size) if mesh_dim is None else int(self.mesh.shape[mesh_dim])

    def get_rank(self):
        return self.rank

    def get_coordinate(self):
        return list(self._coord)

    def ranks_along(self, mesh_dim):
        """Global ranks of the 1-D sub-mesh along `mesh_dim` through my coordinate."""
        idx = list(self._coord)
        idx[mesh_dim] = slice(None)
        return [int(r) for r in self.mesh[tuple(idx)].flatten()]

    def spmd_dims(self):
        dims = [i for i, n in enumerate(self.dim_names) if "spmd" in n]
        return dims if dims else list(range(self.ndim))

    def submesh(self, dims):
        """Mesh over the given dims through my coordinate (e.g. the 'spmd' alias)."""
        idx = [c for c in self._coord]
        for d in dims:
            idx[d] = slice(None)
        return DeviceMesh(self.mesh[tuple(idx)], [self.dim_names[d] for d in dims], self.rank)

    def __repr__(self):
        return f"DeviceMesh({self.mesh.tolist()}, names={self.dim_names}, rank={self.rank})"


_MESH = None


def set_device_mesh(mesh, dim_names=None, rank=None):
    """Accepts an array/list of ranks, a shape TUPLE (ranks 0..n-1 row-major), a torch DeviceMesh or
    the reference's NDDeviceMesh (duck typed: `.mesh` tensor + `.mesh_dim_names`)."""
    global _MESH
    if isinstance(mesh, DeviceMesh):
        _MESH = mesh
        return _MESH
    if hasattr(mesh, "mesh_dim_names") and hasattr(mesh, "mesh"):
        names = dim_names or mesh.mesh_dim_names
        arr = np.asarray(mesh.mesh.cpu().numpy() if hasattr(mesh.mesh, "cpu") else mesh.mesh)
        _MESH = DeviceMesh(arr, names, rank)
        return _MESH
    if isinstance(mesh, tuple) and all(isinstance(v, int) for v in mesh) and \
            dim_names is not None and len(dim_names) == len(mesh):
        arr = np.arange(int(np.prod(mesh))).reshape(mesh)
        _MESH = DeviceMesh(arr, dim_names, rank)
        return _MESH
    _MESH = DeviceMesh(mesh, dim_names, rank)
    return _MESH


def get_device_mesh(alias=None):
    if _MESH is None:
        raise RuntimeError("Device mesh hasn't been set, please call set_device_mesh first.")
    if alias == "spmd":
        dims = _MESH.spmd_dims()
        return _MESH if len(dims) == _MESH.ndim else _MESH.submesh(dims)
    if alias is not None:
        return _MESH.submesh([_MESH.dim_names.index(alias)])
    return _MESH
