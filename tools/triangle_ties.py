#!/usr/bin/env python
"""How many grid points are (numerically) equidistant from two mesh faces, i.e. where the
containing-triangle lookup (utils/legacy/grid_mesh_connectivity.py:89-134: trimesh's
`nearest.on_surface` in the reference, `closest_face_indices` here) has to break a tie.

  python tools/triangle_ties.py > triangle_ties.log
"""
import collections
import os
import sys

import numpy as np
import scipy.spatial

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from graphcast_b200 import grid_mesh_connectivity as gmc, icosahedral_mesh, synthetic   # noqa: E402


def main():
  for res, splits in ((1.0, 5), (0.25, 6)):
    lat, lon = synthetic.grid_coords(res)
    mesh = icosahedral_mesh.get_hierarchy_of_triangular_meshes_for_sphere(splits)[-1]
    pts = gmc._grid_lat_lon_to_coordinates(lat, lon).reshape(-1, 3).astype(np.float64)
    tri = mesh.vertices.astype(np.float64)[mesh.faces]
    tree = scipy.spatial.cKDTree(tri.mean(axis=1))
    gap = np.empty(pts.shape[0])
    for lo in range(0, pts.shape[0], 1 << 15):
      p = pts[lo:lo + (1 << 15)]
      _, cand = tree.query(p, k=8)
      t = tri[cand]
      d2 = np.sort(gmc._point_triangle_sqdist(p[:, None, :], t[:, :, 0], t[:, :, 1], t[:, :, 2]), axis=1)
      gap[lo:lo + p.shape[0]] = d2[:, 1] - d2[:, 0]
    print(f"{res} degree, mesh {splits}: {pts.shape[0]} grid points")
    for eps in (1e-15, 1e-12, 1e-9):
      print(f"  second-closest face within {eps:g} (squared distance) of the closest: {int((gap <= eps).sum())}")
    idx = np.flatnonzero(gap <= 1e-12)
    la = np.repeat(lat, lon.size)[idx]
    lo_ = np.tile(lon, lat.size)[idx]
    print("  of these at the poles:", int((np.abs(la) == 90).sum()), " on the equator:", int((la == 0).sum()))
    c = collections.Counter(np.round(lo_[np.abs(la) < 90], 3).tolist())
    print("  longitudes (count):", c.most_common(8))


if __name__ == "__main__":
  main()
