// per-key comb tables for P-256 (keys grouped inside a launch): construction + fixed-base verification
#include "inst_common.cuh"
using namespace sbv;
const GroupedKtOps sbv_comb_p256 = {{kt_geom<P256, CombTab<P256>>(), op_comb_build<P256>}, op_comb_verify<P256>};
