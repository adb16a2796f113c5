"""Generate tests/golden/labels.npz from the REFERENCE ITSELF: the label rows of label_file_creation.md for seeded poses of
the synthetic closed mesh (synth.closed_mesh), made with utils.py's get_3D_corners and compute_projection, and read back from
a written label file by image.py's fill_truth_detection.

Run where the reference checkout is available (path in REF below):
    python tests/golden/make_golden_labels.py

The rule (label_file_creation.md steps 2-5): the keypoints are the model origin [0, 0, 0] and the 8 get_3D_corners corners;
compute_projection gives their float32 pixel coordinates; a row is [class, x0/w, y0/h, ..., x8/w, y8/h, x range, y range] with
the ranges the width and height of the tight box around the 8 projected corners (step 4), over the image size, in float64.
Stored: the corners (4, 8), K, the poses Rt (n, 3, 4), the projections px (n, 2, 9) float32, the rows (n, 21) float64, and `readback`,
the first row of fill_truth_detection's (50, 21) table for each pose's label file, written by np.savetxt's default format and
read with the identity augmentation (flip 0, dx = dy = 0, sx = sy = 1)."""
import contextlib
import io
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
REF = "/root/reference"
sys.path.insert(0, REPO)

from singleshotpose_b200 import synth          # noqa: E402

W, H, N, CLASS_ID = 640, 480, 16, 3


def main():
    sys.path.insert(0, REF)
    with contextlib.redirect_stdout(io.StringIO()):
        import utils as RU
        import image as RI
    V, F = synth.closed_mesh(seed=1)
    R, t = synth.object_poses(N, seed=7)
    Rt = np.concatenate([R, t[:, :, None]], 2)
    K = synth.intrinsics()
    vertices = np.c_[V, np.ones((len(V), 1))].T
    corners3D = RU.get_3D_corners(vertices)
    P9 = np.concatenate([np.array([[0.0], [0.0], [0.0], [1.0]]), corners3D], 1)
    px, rows, readback = [], [], []
    with tempfile.TemporaryDirectory() as d:
        for p in range(N):
            proj = RU.compute_projection(P9, Rt[p], K)                       # float32 (2, 9)
            x, y = proj[0].astype(np.float64), proj[1].astype(np.float64)
            row = np.r_[CLASS_ID, np.c_[x / W, y / H].reshape(-1), (x[1:].max() - x[1:].min()) / W, (y[1:].max() - y[1:].min()) / H]
            lab = os.path.join(d, "%06d.txt" % p)
            np.savetxt(lab, row[None])
            back = RI.fill_truth_detection(lab, W, H, 0, 0, 0, 1.0, 1.0, 9, 50)
            assert 0 < row[1] < 0.999 and 0 < row[2] < 0.999              # the centroid is inside: no clamp
            px.append(proj); rows.append(row); readback.append(back.reshape(50, 21)[0])
    out = dict(corners3D=corners3D, K=K, Rt=Rt, width=W, height=H, class_id=CLASS_ID, px=np.stack(px), rows=np.stack(rows),
               readback=np.stack(readback))
    assert np.array_equal(out["readback"], out["rows"])
    np.savez_compressed(os.path.join(HERE, "labels.npz"), **out)
    print("labels golden: %d poses, first row %s" % (N, np.round(out["rows"][0], 4).tolist()))


if __name__ == "__main__":
    main()
