// oracle/ref_shims/eigen_digamma.cpp -- TEST INFRASTRUCTURE.  Five lines of glue around the digamma the reference tree
// vendors (include/eigen3/unsupported/Eigen/src/SpecialFunctions/SpecialFunctionsImpl.h, Cephes-derived; SURVEY.md 8c
// names it as the second in-tree reference for boost::math::digamma, which is absent here).  Compiled by
// oracle/build_ref.sh against the headers where they lie in a salmon source tree; nothing of them is copied.
#include <unsupported/Eigen/SpecialFunctions>
extern "C" void ref_eigen_digamma(unsigned long n, const double* x, double* out) {
  for (unsigned long i = 0; i < n; ++i) out[i] = Eigen::numext::digamma(x[i]);
}
