"""Record the golden of the ``--pca`` point colours by running THE REFERENCE'S OWN ``pca_color`` (READ/gl/utils.py:74-91) and the
normalisation of viewer.py:206-209 on seeded descriptors with separated eigenvalues.

Run once where a checkout of the reference exists (READ_REFERENCE_ROOT, default /root/reference) and sklearn is installed; CPU only:

    python tests/golden/make_ref_pca_golden.py

``READ.gl.utils`` is imported with stub modules for ``cv2``, ``trimesh`` and ``READ.gl.programs`` (OpenGL), none of which
``pca_color`` uses, as make_golden.py stubs ``imageio``.  The fixture stores the seed, the point count and the float32 colours.
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.environ.get("READ_REFERENCE_ROOT", "/root/reference"))
for name in ("cv2", "trimesh"):
    sys.modules.setdefault(name, types.ModuleType(name))
programs = types.ModuleType("READ.gl.programs")
programs.NNScene = object
sys.modules.setdefault("READ.gl.programs", programs)

from READ.gl.utils import pca_color                   # noqa: E402

from point_view_util import separated_descriptors     # noqa: E402

SEED, N = 7, 20_000


def main():
    tex = torch.from_numpy(separated_descriptors(N, SEED))
    pca = pca_color(tex)                                               # viewer.py:206
    pca = (pca - np.percentile(pca, 10)) / (np.percentile(pca, 90) - np.percentile(pca, 10))
    pca = np.clip(pca, 0, 1)
    np.savez_compressed(os.path.join(HERE, "ref_pca.npz"), seed=SEED, n=N, colors=pca.astype(np.float32))
    print(f"ref_pca.npz: {N} points, seed {SEED}")


if __name__ == "__main__":
    main()
