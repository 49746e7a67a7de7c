"""CPU twins of tests/test_gpu_mode_transitions.py: the same test functions on the emulated kernels
(tests/test_emu_engine.py explains the emulation and what it does and does not prove)."""
import pytest

import port
from test_emu_engine import emulated_engine  # noqa: F401  (module fixture: the engine library is the emulator build)

pytestmark = pytest.mark.skipif(not port.available(), reason="oracle/_ref/liboracle.so not built")

import test_gpu_mode_transitions as _trans    # noqa: E402

# sync losses while P3 / P4 frames flow, service-mode changes in one stream, decode groups enabled mid-run
test_sync_loss_while_px_frames_flow = _trans.test_sync_loss_while_px_frames_flow
test_mode_chain_in_one_stream = _trans.test_mode_chain_in_one_stream
test_decode_groups_enabled_mid_run = _trans.test_decode_groups_enabled_mid_run
test_sync_loss_with_l2_on_device = _trans.test_sync_loss_with_l2_on_device
test_mode_chain_across_dropouts = _trans.test_mode_chain_across_dropouts
test_am_mode_changes_after_sync_loss = _trans.test_am_mode_changes_after_sync_loss
test_am_rdbi_set = _trans.test_am_rdbi_set
test_psmi_aliases = _trans.test_psmi_aliases
test_psmi_beyond_the_vote_never_acquires = _trans.test_psmi_beyond_the_vote_never_acquires
