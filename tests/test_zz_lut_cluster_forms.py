"""Both forms of the cluster LUT GEMV, forced in turn (runs last: `zz`).  See csrc/gemv_lut.cuh and csrc/capi.cu."""
import pytest
import torch
from helpers import TOL_FP16_TIGHT, c_oracle_check, gpu_case

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("form", ["1", "2", "3", "2-rb32"])
@pytest.mark.parametrize("K", [1, 2])
@pytest.mark.parametrize("fin,fout", [(4096, 4096), (4096, 12288), (4096, 22016), (1024, 200)])
def test_lut_cluster_kernel_forms(form, K, fin, fout, monkeypatch):
    """The cluster LUT GEMV has two forms (csrc/gemv_lut.cuh); the automatic choice (AQLM_B200_LUT_CLUSTER=3, the default)
    is the second form with 16-row warp batches.  Force each (1: first, 2: second, 2-rb32: second with 32-row warp
    batches) so that every one is checked on whatever box runs this, on row blocks of 32 .. 1400 rows (one warp round and
    several), all rows against the C oracle."""
    from aqlm_b200 import _cabi
    from aqlm_b200.inference_kernels import cuda_kernel

    monkeypatch.setenv("AQLM_B200_LUT_CLUSTER", form.split("-")[0])
    if form.endswith("rb32"):
        monkeypatch.setenv("AQLM_B200_LUT_C2_RB", "32")
    _cabi.reload_tunables()  # the switches are cached per process
    try:
        t = gpu_case(fin, fout, K, 8, 1, seed=K * 77 + fin + fout, bias=True)
        y = cuda_kernel.matmat(t["x"], t["codes"], t["codebooks"], t["scales"], t["bias"])
        rel = c_oracle_check(t, y)
        assert rel < TOL_FP16_TIGHT, rel
        y2 = cuda_kernel.matmat(t["x"], t["codes"], t["codebooks"], t["scales"], t["bias"])
        assert torch.equal(y, y2)  # fixed-order cross-slab sum
    finally:
        monkeypatch.delenv("AQLM_B200_LUT_CLUSTER", raising=False)
        monkeypatch.delenv("AQLM_B200_LUT_C2_RB", raising=False)
        _cabi.reload_tunables()
