"""CPU twins of tests/test_gpu_acquisition.py: the same test functions on the emulated kernels
(tests/test_emu_engine.py explains the emulation and what it does and does not prove)."""
import pytest

import port
from test_emu_engine import emulated_engine  # noqa: F401  (module fixture: the engine library is the emulator build)

pytestmark = pytest.mark.skipif(not port.available(), reason="oracle/_ref/liboracle.so not built")

import test_gpu_acquisition as _acq    # noqa: E402

test_cfo_search_winner_off_its_first_trial = _acq.test_cfo_search_winner_off_its_first_trial
test_cfo_search_winner_in_noise = _acq.test_cfo_search_winner_in_noise
test_cfo_search_runs_out = _acq.test_cfo_search_runs_out
test_acquisition_with_short_lead_in = _acq.test_acquisition_with_short_lead_in
