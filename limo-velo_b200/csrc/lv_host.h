/*
 * lv_host.h — host-side pieces of the Localizator / Mapper modules that stay on the CPU in the
 * product (as they do in the reference) and helpers shared by the translation units.
 */
#ifndef LV_HOST_H_
#define LV_HOST_H_

#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "../../include/limovelo_b200.h"

/* Localizator::init_IKFoM_state (src/Modules/Localizator.cpp:135-153) */
void lvh_init_state(const lv_params& prm, const float q_imu[4], double* x, double* P);
/* Localizator::propagate -> esekf::predict (Localizator.cpp:159-173, esekfom.hpp:279-384) */
void lvh_predict(const lv_params& prm, const double acc[3], const double gyro[3], double dt, double* x, double* P);
/* the text lv_last_error() returns (this thread) */
void lvh_set_error(const char* msg);

#endif
