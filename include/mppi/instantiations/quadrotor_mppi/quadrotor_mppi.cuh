// Source-compatibility forwarder: the reference's include path, served by the mppi_b200 host layer.
// With -DMPPIB_USE_INSTANTIATION_LIBRARY the controller classes the reference pre-builds in src/controllers/quadrotor/ are
// declared `extern template` here and come from libmppi_b200_controllers.so (src/controllers/build.sh) instead of being
// instantiated in the including translation unit — the role of the reference's instantiation libraries
// (src/controllers/quadrotor/quadrotor_mppi.cu:3-8: the quadratic-cost and the map-cost controllers). Without the macro everything
// stays header-only (g++ compiles a controller in ~2 s).
#pragma once
#include <mppi/feedback_controllers/DDP/ddp.cuh>
#include <mppi_b200/controllers/MPPI/mppi_controller.hpp>
#include <mppi_b200/cost_functions/quadrotor/quadrotor_map_cost.hpp>
#include <mppi_b200/cost_functions/quadrotor/quadrotor_quadratic_cost.hpp>
#include <mppi_b200/dynamics/quadrotor/quadrotor_dynamics.hpp>

#if defined(MPPIB_USE_INSTANTIATION_LIBRARY) && !defined(MPPIB_INSTANTIATIONS_BUILD)
#define MPPIB_INST extern template class
#elif defined(MPPIB_INSTANTIATIONS_BUILD)
#define MPPIB_INST template class
#endif
#ifdef MPPIB_INST
MPPIB_INST VanillaMPPIController<QuadrotorDynamics, QuadrotorQuadraticCost, DDPFeedback<QuadrotorDynamics, 100>, 100, 512>;
MPPIB_INST VanillaMPPIController<QuadrotorDynamics, QuadrotorMapCost, DDPFeedback<QuadrotorDynamics, 100>, 100, 512>;
#undef MPPIB_INST
#endif
