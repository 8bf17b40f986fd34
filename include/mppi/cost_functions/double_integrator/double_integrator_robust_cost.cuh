// Source-compatibility forwarder: the reference's include path, served by the mppi_b200 host layer.
#pragma once
#include <mppi_b200/cost_functions/double_integrator/double_integrator_robust_cost.hpp>
