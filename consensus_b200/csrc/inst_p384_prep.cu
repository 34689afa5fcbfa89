// prep + key grouping + key cache + G table for P-384
#include "inst_common.cuh"
using namespace sbv;
const CurveOps sbv_ops_p384 = {P384::N, P384::BYTES, (size_t)P384::GWINS << P384::GW, op_gtable_init<P384>, op_prep<P384>, op_route, op_gpart<P384>,
                                sbv_coz_p384, &sbv_kt5_p384, &sbv_kt8_p384};
const GroupOps sbv_group_p384 = {&sbv_kt5_p384, KcXY<P384>::W, 4, op_group<P384>, op_kc_lookup<P384>, op_kc_insert<P384>,
                                 op_kca_lookup<P384>, op_kca_insert<P384>};
