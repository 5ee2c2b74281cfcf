"""CPU: the runtime options of bicg_set_option.  Every option is set with and without its BICG_ prefix; retired experiment
switches are unknown keys."""
import pytest

# every option with its default: setting a key to its default leaves the process's configuration as it was
DEFAULTS = {
    "TOL": "1e-15", "MAX_ITER": "1000", "OUT_ITER": "100", "QUIET": "0",
    "SPMV": "auto", "SPMV_LANES": "0", "SPMV_THREADS": "0", "SPMV_STAGES": "0", "SPMV_CTAS": "0",
    "AUTOTUNE": "1", "UNROLL": "10", "CACHE": "1",
    "MEGA": "1", "MEGA_THREADS": "0", "MEGA_TRACE": "0", "MEGA_LANES": "0", "RESIDENT": "1",
    "BOUNDARY_WEIGHT": "300", "ROW_WEIGHT": "1200", "DEVICE": "-1", "HALO_GAP": "64", "VERBOSE": "0",
    "PEER_TIMEOUT_S": "20", "SHIFT_TOL": "1e-12", "SHIFT_MAX_ITER": "1000", "SHIFT_ERROR": "0",
}
RETIRED = ["GATHER_CG", "L2_HINT", "FENCE_WRITERS", "STAGE_UPLOAD", "GRAPH"]


@pytest.mark.parametrize("prefix", ["", "BICG_"])
def test_every_option_is_known(B, prefix):
    for key, value in DEFAULTS.items():
        assert B.lib.bicg_set_option((prefix + key).encode(), value.encode()) == 0, prefix + key


@pytest.mark.parametrize("key", RETIRED)
@pytest.mark.parametrize("prefix", ["", "BICG_"])
def test_retired_options_are_unknown(B, prefix, key):
    assert B.lib.bicg_set_option((prefix + key).encode(), b"1") == -1
    with pytest.raises(KeyError):
        B.set_option(prefix + key, 1)
