// per-key tables with 8-bit signed windows for registered P-256 keys: construction + fixed-base verification
#include "inst_common.cuh"
using namespace sbv;
const RegisteredKtOps sbv_kt8_p256 = {{kt_geom<P256, KeyTab<256, 8>>(), op_kt_build<P256, 8>}, op_kt_verify_registered<P256, 8>};
