// Explicit instantiations of the controller classes the reference pre-builds in src/controllers/quadrotor/quadrotor_mppi.cu (the
// quadratic-cost and the map-cost VanillaMPPIController), as plain host C++ (the device code lives behind the C ABI in
// libmppi_b200.so): built into libmppi_b200_controllers.so by
// src/controllers/build.sh; users that define MPPIB_USE_INSTANTIATION_LIBRARY get `extern template` declarations instead.
#define MPPIB_INSTANTIATIONS_BUILD
#include <mppi/instantiations/quadrotor_mppi/quadrotor_mppi.cuh>
