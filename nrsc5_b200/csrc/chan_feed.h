// The seam between the wideband channeliser (channelizer.cu) and the receive engine (engine.cu) behind
// nrsc5b_chan_feed.  Not part of the C ABI.  Neither side sees the other's struct: the channeliser asks the engine for
// room and for where each target stream's next cs16 sample goes, launches its kernel on the engine's CUDA stream, and
// then tells the engine how many samples it wrote into every target stream.
#ifndef NRSC5_B200_CHAN_FEED_H
#define NRSC5_B200_CHAN_FEED_H

#include <cuda_runtime.h>

#include "../../include/nrsc5_b200.h"

struct FeedTarget {
    cudaStream_t stream;       // the engine's CUDA stream: the feed runs on it
    int16_t *base;             // the engine's own input buffers; dst[k] below counts int16 values from here
};

// Checks that `e` can take nch channels into `streams` (NULL: stream k for channel k) from a channeliser on `device`
// whose band plan makes channels for engines of `mode` (NRSC5B_MODE_FM | NRSC5B_MODE_AM), and makes room for nout cs16 samples in each target stream (a full stream is trimmed first, as the pushes do: the
// samples its receiver has moved past are dropped).  dst[k] = where channel k's first sample goes.
//   NRSC5B_EINVAL: not an engine of that mode reading its own cs16 input buffers, another device, an asynchronous batch in
//                  flight, or stream indices repeated or out of range;
//   NRSC5B_EFULL:  some target stream has no room for nout samples even after trimming.
// Nothing but those trims has happened when it returns an error.
int nbfeed_reserve(nrsc5b_engine_t *e, int device, int mode, const int *streams, int nch, long long nout, FeedTarget *t, long long *dst);

// nout samples have been written (stream-ordered on t.stream) behind every target stream's data: count them and
// publish the new sample counts to the kernels after the writes.
int nbfeed_commit(nrsc5b_engine_t *e, const int *streams, int nch, long long nout);

#endif
