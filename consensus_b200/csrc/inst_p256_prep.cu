// prep + key grouping + key cache + G table for P-256
#include "inst_common.cuh"
using namespace sbv;
const CurveOps sbv_ops_p256 = {P256::N, P256::BYTES, (size_t)P256::GWINS << P256::GW, op_gtable_init<P256>, op_prep<P256>, op_route, op_gpart<P256>,
                                sbv_coz_p256, &sbv_comb_p256, &sbv_kt8_p256};
const GroupOps sbv_group_p256 = {&sbv_comb_p256, KcXY<P256>::W, 5, op_group<P256>, op_kc_lookup<P256>, op_kc_insert<P256>,
                                 op_kca_lookup<P256>, op_kca_insert<P256>};
