// hb_dist.h — point-to-point exchange primitive used by the row-sharded local_laplacian (implemented in hb_dist.cu).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

namespace hbdist {

struct Msg {
    void *ptr;     // device address
    size_t bytes;
    int peer;      // rank
    bool send;     // true: ncclSend, false: ncclRecv
};

bool active();
int rank();
int size();
// Changes whenever the calling thread joins a communicator: state kept per geometry is only valid within one.
int epoch();
// One ncclGroup of point-to-point messages enqueued on stream `s` (ordered with the kernels on it).
int exchange(const Msg *msgs, int n, cudaStream_t s);

// Host-side all-gather of a small POD blob (plan setup only, synchronous): recv_all holds size() blobs in rank order.
int allgather_bytes(const void *send, void *recv_all, size_t bytes_per_rank);

}  // namespace hbdist
