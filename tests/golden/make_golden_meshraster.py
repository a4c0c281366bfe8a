"""Golden mesh for the mesh-render tests: the reference's low-poly human (load/shapes/human.obj), fan-triangulated.

The OBJ has 1 629 vertices and 1 694 polygons (212 triangles, 1 432 quads and 50 pentagons); polygon (p0, ..., pn-1)
becomes the triangles (p0, pk, pk+1), k = 1..n-2, in file order: 3 226 triangles.  Writes ref_meshraster.npz
(vertices [1629, 3] float32, faces [3226, 3] int32).  This is a data fixture only; the tests do not need the reference.

    HUMANGAUSSIAN_ROOT=<reference checkout> python tests/golden/make_golden_meshraster.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import meshraster_reference as M  # noqa: E402

REF = os.environ["HUMANGAUSSIAN_ROOT"]


def main():
    verts, polys = M.load_obj_polygons(os.path.join(REF, "load", "shapes", "human.obj"))
    sizes = np.bincount([len(p) for p in polys])
    assert verts.shape == (1629, 3) and len(polys) == 1694 and tuple(sizes[3:6]) == (212, 1432, 50), (verts.shape, sizes)
    faces = M.fan_triangulate(polys)
    assert faces.shape == (3226, 3) and faces.min() >= 0 and faces.max() < len(verts)
    np.savez_compressed(M.GOLDEN, vertices=verts, faces=faces)
    print(f"wrote {M.GOLDEN}: {len(verts)} vertices, {len(faces)} triangles")


if __name__ == "__main__":
    main()
