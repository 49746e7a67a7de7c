"""CPU: the oracle (oracle/nrsc5_oracle*.c, what the GPU tests compare against) equals the unmodified reference on
the captures of tests/test_gpu_mode_transitions.py - sync losses while P3 / P4 frames flow, a stream that changes
service mode between acquisitions, AM mode changes, PSMI aliases - so that the restatement is pinned where the
receiver's state carries over from one mode to the next."""
import pytest

import common
import mode_transitions as mt
import port
import reftap

pytestmark = pytest.mark.skipif(not (reftap.available() and port.available()), reason="oracle/_ref/ not built")


def _same(samples, mode=reftap.MODE_FM):
    a = port.decode(samples) if mode == reftap.MODE_FM else port.decode_am(samples)
    b = reftap.decode(samples, mode=mode)
    assert common.summarize(a) == common.summarize(b)
    return [e[0] for e in common.summarize(b)]


@pytest.mark.parametrize("name", list(mt.LOSS_CASES))
def test_oracle_sync_loss_while_px_frames_flow(name):
    kinds = _same(mt.cu8_of([mt.loss_capture(name)]))
    assert "L" in kinds


@pytest.mark.parametrize("gaps", [False, True])
def test_oracle_mode_chain(gaps):
    kinds = _same(mt.chain_capture(gaps))
    assert kinds.count("S") >= 5 and kinds.count("L") >= 4


def test_oracle_am_mode_chain():
    assert _same(mt.am_chain(), reftap.MODE_AM).count("L") >= 2


@pytest.mark.parametrize("psmi", [1, 2])
def test_oracle_am_rdbi(psmi):
    assert "F" in _same(mt.am_rdbi(psmi), reftap.MODE_AM)


@pytest.mark.parametrize("psmi", mt.ALIASES + [mt.NEVER])
def test_oracle_psmi_aliases(psmi):
    kinds = _same(mt.alias_capture(psmi))
    assert ("S" in kinds) == (psmi < 16)
