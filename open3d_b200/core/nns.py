"""``open3d.core.nns.NearestNeighborSearch`` on the device (core/nns/NearestNeighborSearch.h): the exact k-nearest-
neighbour search (o3db_knn_*) and the hybrid search (o3db_nns_*).  Fixed-radius and multi-radius search are not built
(DESIGN.md §7)."""
from __future__ import annotations

import ctypes as C

import torch

from .._lib import INDEX_INT32, INDEX_INT64, check, lib
from . import as_device_f32_points, current_stream_ptr


class _Handle:
    """Owns one C-ABI index handle and destroys it with its destroy function."""

    def __init__(self, destroy):
        self.ptr = C.c_void_p()
        self._destroy = destroy

    def __del__(self):
        if self.ptr:
            self._destroy(self.ptr)
            self.ptr = C.c_void_p()


class NearestNeighborSearch:
    """core::nns::NearestNeighborSearch over an [M, 3] Float32 dataset.  Indices come back in ``index_dtype``
    (torch.int32 or torch.int64); every result stays on the device."""

    def __init__(self, dataset_points, index_dtype=torch.int64):
        if index_dtype not in (torch.int32, torch.int64):
            raise RuntimeError(f"index_dtype must be torch.int32 or torch.int64, got {index_dtype}")
        self.dataset_points = as_device_f32_points(dataset_points, "dataset_points")
        self.index_dtype = index_dtype
        self._knn = None
        self._hybrid = None
        self._hybrid_radius = None

    def knn_index(self):
        """NearestNeighborSearch::KnnIndex: builds the exact KNN index; True on success."""
        h = _Handle(lib.o3db_knn_destroy)
        p = self.dataset_points
        check(lib.o3db_knn_create(p.data_ptr(), int(p.shape[0]), current_stream_ptr(), C.byref(h.ptr)))
        self._knn = h
        return True

    def knn_search(self, query_points, knn):
        """NearestNeighborSearch::KnnSearch -> (indices [Q, k'], squared distances [Q, k']), k' = min(knn, M),
        ascending by distance, ties to the lower index; knn in 1..32.  A query with a non-finite coordinate gets a
        row of -1 and 0."""
        if self._knn is None:
            raise RuntimeError("Index is not set.")
        q = as_device_f32_points(query_points, "query_points")
        knn = int(knn)
        nq = int(q.shape[0])
        kp = max(0, min(knn, int(self.dataset_points.shape[0])))
        idx = torch.empty((nq, kp), dtype=self.index_dtype, device=q.device)
        dist = torch.empty((nq, kp), dtype=torch.float32, device=q.device)
        check(lib.o3db_knn_search(self._knn.ptr, q.data_ptr(), nq, knn,
                                  INDEX_INT64 if self.index_dtype == torch.int64 else INDEX_INT32, idx.data_ptr(),
                                  dist.data_ptr(), current_stream_ptr()))
        return idx, dist

    def hybrid_index(self, radius):
        """NearestNeighborSearch::HybridIndex(radius); True on success."""
        h = _Handle(lib.o3db_nns_destroy)
        p = self.dataset_points
        check(lib.o3db_nns_create(p.data_ptr(), int(p.shape[0]), float(radius), current_stream_ptr(), C.byref(h.ptr)))
        self._hybrid = h
        self._hybrid_radius = float(radius)
        return True

    def hybrid_search(self, query_points, radius, max_knn):
        """NearestNeighborSearch::HybridSearch -> (indices [Q, max_knn], squared distances [Q, max_knn], counts [Q]):
        up to max_knn (1..32) nearest points within radius, padded with -1 and 0."""
        if self._hybrid is None:
            raise RuntimeError("Index is not set.")
        q = as_device_f32_points(query_points, "query_points")
        nq, max_knn = int(q.shape[0]), int(max_knn)
        k = max(max_knn, 0)
        idx = torch.empty((nq, k), dtype=torch.int32, device=q.device)
        dist = torch.empty((nq, k), dtype=torch.float32, device=q.device)
        cnt = torch.empty((nq,), dtype=torch.int32, device=q.device)
        check(lib.o3db_nns_hybrid_search(self._hybrid.ptr, q.data_ptr(), nq, float(radius), max_knn, idx.data_ptr(),
                                         dist.data_ptr(), cnt.data_ptr(), current_stream_ptr()))
        return idx.to(self.index_dtype), dist, cnt.to(self.index_dtype)

    def _not_built(self, *args, **kwargs):
        raise RuntimeError("fixed-radius and multi-radius search are not built in open3d_b200 (DESIGN.md §7); use "
                           "knn_search or hybrid_search")

    fixed_radius_index = fixed_radius_search = multi_radius_index = multi_radius_search = _not_built
