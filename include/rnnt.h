/* include/rnnt.h -- C ABI of the RNN-T loss library, binary-compatible with the one the
 * reference vendors (warp-transducer/include/rnnt.h:1-147 @ f546575): same symbol names,
 * argument order, enum values and by-value options struct, so bindings written against
 * libwarprnnt.so (pytorch_binding/src/binding.cpp:84-154, tensorflow_binding/src/warprnnt_op.cc)
 * load libedgedict_b200.so unchanged.
 *
 * Differences in behaviour (documented in INTEGRATION.md):
 *   - only RNNT_GPU is implemented (sm_90a); RNNT_CPU returns RNNT_STATUS_EXECUTION_FAILED;
 *   - get_workspace_size() reports this library's own requirement (5*T*U+2 scalars per
 *     utterance); callers already size the workspace through it;
 *   - as in the reference's GPU path, activations are raw logits, labels / lengths / workspace
 *     are DEVICE pointers and costs is a HOST pointer (the call synchronises the stream once).
 */
#pragma once
#ifdef __cplusplus
#include <cstddef>
extern "C" {
#else
#include <stddef.h>
#include <stdbool.h>
#endif

typedef struct CUstream_st* CUstream;

typedef enum {
    RNNT_STATUS_SUCCESS = 0,
    RNNT_STATUS_MEMOPS_FAILED = 1,
    RNNT_STATUS_INVALID_VALUE = 2,
    RNNT_STATUS_EXECUTION_FAILED = 3,
    RNNT_STATUS_UNKNOWN_ERROR = 4
} rnntStatus_t;

typedef enum { RNNT_CPU = 0, RNNT_GPU = 1 } rnntComputeLocation;

struct rnntOptions {
    rnntComputeLocation loc;  /* must be RNNT_GPU                                   */
    unsigned int num_threads; /* ignored (CPU-only knob of the reference)           */
    CUstream stream;          /* all kernels are enqueued here                      */
    int blank_label;
    int maxT;                 /* padded time length of the acts tensor              */
    int maxU;                 /* padded label length + 1                            */
    bool batch_first;         /* layout is always (b, t, u, v) row-major            */
};
#ifndef __cplusplus
typedef struct rnntOptions rnntOptions;
#endif

int get_warprnnt_version(void);
const char* rnntGetStatusString(rnntStatus_t status);

/* acts[((b*maxT + t)*maxU + u)*V + v]; gradients may be NULL (forward score only);
 * flat_labels has row stride maxU-1. */
rnntStatus_t compute_rnnt_loss(const float* const activations, float* gradients,
                               const int* const flat_labels, const int* const label_lengths,
                               const int* const input_lengths, int alphabet_size, int minibatch,
                               float* costs, void* workspace, struct rnntOptions options);

rnntStatus_t compute_rnnt_loss_fp64(const double* const activations, double* gradients,
                                    const int* const flat_labels, const int* const label_lengths,
                                    const int* const input_lengths, int alphabet_size,
                                    int minibatch, double* costs, void* workspace,
                                    struct rnntOptions options);

rnntStatus_t get_workspace_size(int maxT, int maxU, int minibatch, bool gpu, size_t* size_bytes,
                                size_t dtype_size
#ifdef __cplusplus
                                = sizeof(float)
#endif
);

#ifdef __cplusplus
}
#endif
