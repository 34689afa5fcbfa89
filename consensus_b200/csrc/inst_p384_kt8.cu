// per-key tables with 8-bit signed windows for P-384: construction + fixed-base verification
#include "inst_common.cuh"
using namespace sbv;
const KtOps sbv_kt8_p384 = {kt_geom<P384, KeyTab<384, 8>>(), op_kt_build<P384, 8>, op_kt_verify<P384, 8>};
