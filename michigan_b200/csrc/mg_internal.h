// michigan_b200 — internal helpers shared by the translation units of libmichigan_sm90.so.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include "../../include/michigan_b200.h"

namespace mg {

// printf-style; stores the message in a thread-local buffer and returns `code`.
int set_error(int code, const char* fmt, ...);
void count_launch(int n = 1);
int num_sms();
// cuTensorMapEncodeTiled through the runtime's driver entry point (no link against libcuda).
int encode_tensor_map(CUtensorMap* map, void* gaddr, CUtensorMapDataType dtype, int rank, const cuuint64_t* dims, const cuuint64_t* strides,
                      const cuuint32_t* box, const cuuint32_t* estrides, CUtensorMapSwizzle swizzle);

// Tuning knobs (alternative schedules that all give the same results): read ONCE from the environment at first use,
// overridable through mg_set_tuning() (tests, A/B tools).  Nothing on the launch path calls getenv.
enum TuneKnob {
    TK_MERGE = 0,        // MG_MERGE: split-precision convs with 2*BN <= 128 as two MMAs per K step (default 1)
    TK_HALO,             // MG_HALO: halo schedule of 3x3/s1 convs (default 0)
    TK_HALO_PW,          // MG_HALO_PW: patch pitch 10 | 16
    TK_EPI_IMPL,         // MG_EPI_IMPL: 1 transposed epilogue (default), 0 row-per-lane reference epilogue
    TK_EPI_IMPL_SPADE,   // MG_EPI_IMPL_SPADE (default: = MG_EPI_IMPL)
    TK_EPI_CW16,         // MG_EPI_CW16: 16-channel epilogue chunks (default 1)
    TK_CW_SPADE,         // MG_EPI_CW_SPADE: 16 | 32
    TK_STAGES,           // MG_STAGES: cap on the smem ring depth (0 = none)
    TK_THIN_GEMM,        // MG_THIN_GEMM (default 1)
    TK_GROUP3,           // MG_GROUP3: 3x3/s1 convs on the halo-patch + M-tile-group kernel (mg_conv3x3.cu): 0 off, 1 / 2 on
    TK_SEG_TMA,          // MG_SEG_TMA: 16-bit outputs of the seg conv through smem staging + TMA stores (default 1)
    TK_BN_FILL,          // MG_BN_FILL: generic convs whose tiles do not fill the SMs use a narrower BN (default 1)
    TK_EPI_REG,          // MG_EPI_REG: epilogue of the 3x3 group kernel on the accumulator registers (default 1), 0 through smem
    TK_COUNT
};
int tune(int knob);

// What-if probes (skip loads / epilogue work: WRONG results, timing experiments only) and the clock64() role profile exist
// only in a library built with -DMG_PROBES (python -m michigan_b200.build --probes -> libmichigan_sm90_probes.so);
// the product library compiles them out.
#ifdef MG_PROBES
int probe_bits();   // env MG_DBG, read once
#define MG_DBGV(p) ((p).dbg)
#define MG_PROFV(p) ((p).prof)
#else
#define MG_DBGV(p) 0
#define MG_PROFV(p) 0
#endif

// mg_orient.cu: mg_conv_thin with argmax_idx set (the DoG orientation response and its batch maximum)
int orient_argmax_conv(const mg_thin_args* a, cudaStream_t stream);

struct IgemmParams;
// mg_conv3x3.cu: 1 = launched, 0 = shape not eligible (use the per-tap kernel), anything else = error status
int conv3x3_group_launch(const mg_igemm_args* a, IgemmParams& p, int BN, int cw, int scratch_bytes, int spec, cudaStream_t stream);

// Order-independent reductions.  Kernels whose CTAs add partial sums into the same elements in whatever order they finish
// accumulate into a zeroed fp64 buffer instead of the fp32 destination: sums of fp32 partials of the magnitudes met here are
// exact in fp64, so the result no longer depends on the finishing order and two runs on the same inputs agree bit for bit.
// acc64_fold then writes dst[i] = (add ? dst[i] : 0) + (float)acc[i].  All three are stream-ordered.
int acc64_alloc(double** acc, size_t n, cudaStream_t stream);
int acc64_fold(const double* acc, float* dst, size_t n, int add, cudaStream_t stream);
int acc64_free(double* acc, cudaStream_t stream);

inline int check_launch(const char* what) {
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_error((int)e, "%s: %s", what, cudaGetErrorString(e));
    return 0;
}

}  // namespace mg
