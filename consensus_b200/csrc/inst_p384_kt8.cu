// per-key tables with 8-bit signed windows for registered P-384 keys: construction + fixed-base verification
#include "inst_common.cuh"
using namespace sbv;
const RegisteredKtOps sbv_kt8_p384 = {{kt_geom<P384, KeyTab<384, 8>>(), op_kt_build<P384, 8>}, op_kt_verify_registered<P384, 8>};
