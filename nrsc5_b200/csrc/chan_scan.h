// What nrsc5b_chan_scan (scan.cu) needs to know of a channeliser handle (channelizer.cu), whose struct it does not see.
// Not part of the C ABI.
#ifndef NRSC5_B200_CHAN_SCAN_H
#define NRSC5_B200_CHAN_SCAN_H

#include "../../include/nrsc5_b200.h"

// the handle's device, the engine mode its plan makes channels for (NRSC5B_MODE_FM | NRSC5B_MODE_AM), its input format
// (1: cs16) and its channel count
int nbchan_info(const nrsc5b_channelizer_t *c, int *device, int *mode, int *cs16, int *nch);

// outputs per channel that a push of `samples` more complex samples would emit now
long long nbchan_outputs_after(const nrsc5b_channelizer_t *c, long long samples);

#endif
