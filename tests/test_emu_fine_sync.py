"""CPU twins of tests/test_gpu_fine_sync.py: the same test functions on the emulated kernels
(tests/test_emu_engine.py explains the emulation and what it does and does not prove)."""
import pytest

import port
from test_emu_engine import emulated_engine  # noqa: F401  (module fixture: the engine library is the emulator build)

pytestmark = pytest.mark.skipif(not port.available(), reason="oracle/_ref/liboracle.so not built")

import test_gpu_fine_sync as _fs    # noqa: E402

test_multi_stream_mp1_soft_bits_mer_and_pdus = _fs.test_multi_stream_mp1_soft_bits_mer_and_pdus
test_extended_partitions = _fs.test_extended_partitions
test_cfo_search_then_fine_sync = _fs.test_cfo_search_then_fine_sync
