"""GPU: the plane GEMM's 120- and 240-column tiles (gcc-nmf_b200/csrc/tma_gemm.cuh) against a float64 product.  On a 132-SM
H100 the KL-NMF planner runs the W.H contractions on 120-column dual-N tiles (wgmma of N = 120 and N = 240 per k-step) and the
H update on plain 240-column tiles (three wgmma of N = 240)."""
import pytest

from test_gpu_tma import _gemm_error

pytestmark = pytest.mark.gpu

# (M, N, Kc): one ragged tile; the 513-row SIMT tail with several n tiles; the k tail and a ragged n tile
SHAPES = [(128, 120, 64), (513, 640, 256), (256, 416, 513)]
SHAPES_240 = [(128, 240, 64), (513, 640, 256), (256, 513, 1024)]


@pytest.fixture(scope='module')
def h():
    from gcc_nmf_b200._lib import default_handle
    return default_handle()


def test_plane_gemm_dual_n_120(h):
    """120-column dual-N tiles (A_lo . B_hi of N = 120, A_hi . [B_hi; B_lo] of N = 240 per k-step): K-major B, both A layouts."""
    for M, N, Kc in SHAPES:
        for a_mn in (False, True):
            err = _gemm_error(h, M, N, Kc, a_mn, False, 120, 1)
            assert err < 8e-6 + 4e-8 * (3 * Kc / 16), ((M, N, Kc), a_mn, err)


def test_plane_gemm_plain_240(h):
    """240-column tiles, three wgmma of N = 240 per k-step: B K-major and MN-major (a K-major A with a K-major B as well)."""
    for M, N, Kc in SHAPES_240:
        for a_mn, b_mn in ((False, False), (True, False), (True, True)):
            err = _gemm_error(h, M, N, Kc, a_mn, b_mn, 240, 1)
            assert err < 8e-6 + 4e-8 * (3 * Kc / 16), ((M, N, Kc), (a_mn, b_mn), err)


def test_plane_gemm_120_is_dual_n_only(h):
    """120 columns are instantiated for the dual-N loop only: an MN-major B operand is refused, not run on a wrong kernel."""
    import torch
    from gcc_nmf_b200._lib import GCCNMFError
    A = torch.rand(64, 128, device=h.device)
    B = torch.rand(64, 120, device=h.device)
    with pytest.raises(GCCNMFError):
        h.gemm_planes(A, B, True, True, tile_n=120)
