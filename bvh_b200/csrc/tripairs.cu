// bvh_b200/csrc/tripairs.cu -- the triangle-pair walks of csr.cuh (bvhgpu_triangle_pairs_*) with the exact predicate of tritri.cuh,
// over Tree<T> (D = 3).  A translation unit of their own, so that the predicate and its exact fallbacks are compiled once.
#include "tritri.cuh"
#include "csr.cuh"

namespace bvhb200 {

template int triangle_pairs_csr<float>(Tree<float>*, int, const CsrOut&, const char*);
template int triangle_pairs_csr<double>(Tree<double>*, int, const CsrOut&, const char*);
template int triangle_pairs_trees_csr<float>(Tree<float>*, Tree<float>*, const CsrOut&, const char*);
template int triangle_pairs_trees_csr<double>(Tree<double>*, Tree<double>*, const CsrOut&, const char*);

}  // namespace bvhb200
