"""mulls_destroy gives back every scratch buffer a context grew, not only the NDT and GICP scratch that
test_gpu_gicp.py checks: creating a context, running each entry point that grows one and closing it, four times, leaves
the device's free memory where it was. At these sizes each round grows about 261 MB of scratch, computed from the
layouts in mulls_b200.cu (not measured): ndt_buf 56 MB, cls_buf 53, gf_buf 32, gicp_buf 32, pca_buf 31, vx_buf 27,
ext_buf 18, raw_buf 11, and under 1 MB each for sor_buf, rc_buf, ncc_buf, nms_buf and gf_cell_buf. A leak would lose
that for the rest of the process."""
import numpy as np
import pytest

from mulls_b200 import abi
from mulls_b200.registration import Context
from test_gicp import LIBC
from test_ncc import kpts
from test_ndt import bbox, structured_scene
from test_rawscan import TRANSFORMS, rows_of, scan_like

pytestmark = pytest.mark.gpu


def test_every_scratch_buffer_released():
    import torch

    tgt = structured_scene(200000, 5)
    src = tgt[::4].copy()
    scene = rows_of(tgt)
    scan = scan_like(200000, np.random.default_rng(1))
    rng = np.random.default_rng(2)
    kt, ks = kpts(2000, rng), kpts(2000, rng)
    gp, cp = abi.default_ground_params(), abi.default_classify_params()

    def once():
        c = Context(0, 2, 250000, 250000)
        try:
            c.pca_features(scan, 1.0, 30)  # pca_buf
            c.pca_features(scan, 1.0, 30, unit_dist=30.0)
            c.sor_filter(scan, 10, 1.0)  # sor_buf
            c.vertical_intrinsic_calibration(scan, 0.5)  # raw_buf
            c.timestamp_ratio(scan, True)
            c.motion_compensation(scan, TRANSFORMS["small"])
            c.ncc_correspondences(kt, ks)  # ncc_buf
            c.ncc_correspondences(kt, ks, True, 2000)
            c.coarse_reg_ransac(kt, ks)  # rc_buf
            c.non_max_suppress(kt, 0.25)  # nms_buf
            c.extract_semantic_pts(scene, 0.1, gp, cp)  # ext_buf, vx_buf, gf_buf, gf_cell_buf, cls_buf
            c.omp_ndt_batch([tgt, tgt], [src, src], [bbox(tgt)] * 2, [bbox(src)] * 2)  # ndt_buf
            c.omp_ndt(tgt, src, bbox(tgt), bbox(src))
            LIBC.srand(1)
            c.omp_gicp(tgt, src, bbox(tgt), bbox(src))  # gicp_buf
        finally:
            c.close()

    once()  # module loading and the runtime's own first allocations
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info(0)[0]
    for _ in range(4):
        once()
    torch.cuda.synchronize()
    free1 = torch.cuda.mem_get_info(0)[0]
    assert free0 - free1 < (32 << 20), (free0 - free1) / 2**20
