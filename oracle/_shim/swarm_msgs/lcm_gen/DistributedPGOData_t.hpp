// Stand-in for the LCM type DistributedPGOData_t (generated, un-vendored), which d2common/d2pgo_types.h names in DPGOData's
// LCM conversions.  The pins never convert: the type only has to exist.
#pragma once
struct DistributedPGOData_t {};
