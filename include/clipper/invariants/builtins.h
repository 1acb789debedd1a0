/** @file builtins.h  (mirror of reference invariants/builtins.h) */
#pragma once
#include "clipper/invariants/euclidean_distance.h"
#include "clipper/invariants/pointnormal_distance.h"
#include "clipper/invariants/cuda_invariant.h"
