"""CPU checks of the partial-buffer sizes the norm backward kernels report (lv_rmsnorm_bwd_partials,
lv_layernorm_bwd_partials).  The caller allocates that many fp32 rows and sums all of them, and the kernel writes one
row per row slot of each CTA, so the size must follow the kernel's row tiling exactly.  The functions need no device:
without one the library assumes 132 SMs."""
import pytest

# threads per row by columns / 8 (the TPR half of each tiling table in csrc/elementwise.cu)
RMSNORM_TPR = ((128, 32), (640, 128), (None, 256))
LAYERNORM_TPR = ((128, 32), (512, 128), (None, 256))


def expected_partials(tpr_table, rows, cols, sms):
    nvec = cols // 8
    tpr = next(t for max_nvec, t in tpr_table if max_nvec is None or nvec <= max_nvec)
    rpc = 256 // tpr
    grid = min(max(-(-rows // rpc), 1), 2 * sms)
    return grid * rpc


def test_the_rule_reproduces_known_sizes():
    assert expected_partials(RMSNORM_TPR, 1000, 5120, 132) == 528
    assert expected_partials(RMSNORM_TPR, 10 ** 6, 8192, 132) == 264
    assert expected_partials(RMSNORM_TPR, 0, 1024, 132) == 8
    assert expected_partials(LAYERNORM_TPR, 10 ** 6, 4096, 132) == 528


@pytest.mark.parametrize("name,tpr_table", [("lv_rmsnorm_bwd_partials", RMSNORM_TPR),
                                            ("lv_layernorm_bwd_partials", LAYERNORM_TPR)])
def test_norm_backward_partials_follow_the_row_tiling(lib_built, name, tpr_table):
    from long_vita_b200 import _lib, ops

    fn = getattr(_lib.lib(), name)
    sms = ops._sm_count(0)
    bad = [(rows, cols, int(fn(rows, cols)), expected_partials(tpr_table, rows, cols, sms))
           for cols in range(8, 16384 + 1, 8) for rows in (0, 1, 7, 255, 1000, 10 ** 6)
           if int(fn(rows, cols)) != expected_partials(tpr_table, rows, cols, sms)]
    assert not bad, f"{name}: (rows, cols, got, want) {bad[:8]}"
