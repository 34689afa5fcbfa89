// per-key tables with 5-bit signed windows for P-384 keys grouped inside a launch: construction + fixed-base verification
#include "inst_common.cuh"
using namespace sbv;
const GroupedKtOps sbv_kt5_p384 = {{kt_geom<P384, KeyTab<384, 5>>(), op_kt_build<P384, 5>}, op_kt_verify_grouped<P384, 5>};
