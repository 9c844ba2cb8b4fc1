// pqp_smoother_internal.h — what other translation units of the library may ask a pqp_smoother_handle
// (defined in pqp_smoother.cu).
#pragma once
#include "../../include/pqp_smoother.h"

namespace pqs {
// NULL if the handle serves the Cartesian tension QP, else why not (its p_max is beyond the QP's shared-memory limit)
const char *cartesian_unavailable(const pqp_smoother_handle *h);
}  // namespace pqs
