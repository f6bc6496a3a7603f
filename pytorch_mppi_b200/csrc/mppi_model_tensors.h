// mppi_model_tensors.h — the device-tensor views of a user model's parameter block (CudaModel(tensors=...)): their
// layout, the checks of the references a caller passes, and the packer.  Plain C++ (no CUDA), so that the layout the
// library packs can be checked on the host against the struct the model header declares (tests/test_model_tensors.py).
//
// The block of a model with n >= 1 tensors is `struct P { real v[NP]; TensorView<T0, N0> t0; ...; }` (the generated
// header, pytorch_mppi_b200/models.py): the views start at the first 8-byte boundary behind the parameters, and every
// view is { const T* data; int shape[4]; } — 24 bytes, 8-aligned, whatever its element type and ndim.
#pragma once
#include <stdint.h>
#include <string.h>

#include "../../include/mppi_b200.h"

namespace mppi_tensors {

struct ViewBytes {
    const void* data;
    int32_t shape[4];
};
static_assert(sizeof(ViewBytes) == 24, "a tensor view is 24 bytes");

inline int views_offset(int np, int real_bytes) { return (np * real_bytes + 7) / 8 * 8; }
inline int block_bytes(int np, int real_bytes, int n) {
    return n > 0 ? views_offset(np, real_bytes) + n * (int)sizeof(ViewBytes) : np * real_bytes;
}
inline bool known_dtype(int32_t dtype) { return dtype == MPPI_F32 || dtype == MPPI_F64 || dtype == MPPI_U8 || dtype == MPPI_I32; }

// MPPI_OK if `refs` (n of them) match a model compiled for (dtypes, ndims) (n_sig of them), else MPPI_ERR_BAD_ARG
inline int check_refs(const int32_t* dtypes, const int32_t* ndims, int n_sig, const MppiTensorRef* refs, int n) {
    if (n != n_sig || (n > 0 && refs == nullptr)) return MPPI_ERR_BAD_ARG;
    for (int i = 0; i < n; ++i) {
        const MppiTensorRef& r = refs[i];
        if (r.data == nullptr || r.dtype != dtypes[i] || r.ndim != ndims[i]) return MPPI_ERR_BAD_ARG;
        int64_t elems = 1;
        for (int d = 0; d < r.ndim; ++d) {
            if (r.shape[d] <= 0 || r.shape[d] > INT32_MAX / elems) return MPPI_ERR_BAD_ARG;   // elems stays <= 2^31 - 1
            elems *= r.shape[d];
        }
    }
    return MPPI_OK;
}

// the views of `refs` (checked) into a parameter block whose parameters are np reals of real_bytes each
inline void pack_views(void* block, int np, int real_bytes, const MppiTensorRef* refs, int n) {
    unsigned char* dst = (unsigned char*)block + views_offset(np, real_bytes);
    for (int i = 0; i < n; ++i) {
        ViewBytes v;
        memset(&v, 0, sizeof(v));
        v.data = refs[i].data;
        for (int d = 0; d < refs[i].ndim; ++d) v.shape[d] = (int32_t)refs[i].shape[d];
        memcpy(dst + i * sizeof(ViewBytes), &v, sizeof(v));
    }
}

}  // namespace mppi_tensors
