// The K per-object map pointers of a merge (DESIGN.md §24), passed by value as a kernel parameter: shared by
// merge_objects_kernel (measures.cu) and upsample_merge_objects_kernel (resize.cu).
#pragma once
#include "common.cuh"

namespace osvos {

struct MergeMaps {
  const float* map[OSVOS_MERGE_MAX_OBJECTS];
};

}  // namespace osvos
