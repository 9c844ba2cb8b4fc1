// pqp_bounds_internal.h — what other translation units of the library may ask a pqp_bounds_handle
// (defined in pqp_bounds.cu): the device-resident map view, the slot table of the per-path maps and the device they
// live on.
#pragma once
#include "../../include/pqp_bounds.h"
#include "pqp_bounds_core.cuh"

namespace pqb {
const MapView *handle_map(const pqp_bounds_handle *h);  // slot 0, the map of the unmapped calls
int handle_device(const pqp_bounds_handle *h);
const MapView *handle_table(const pqp_bounds_handle *h);  // device [handle_map_count] for pqb::slot_view
int handle_map_count(const pqp_bounds_handle *h);
}  // namespace pqb
