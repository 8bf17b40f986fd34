// Source-compatibility forwarder: the reference's include path, served by the mppi_b200 host layer.
#pragma once
#include <mppi_b200/sampling_distributions/smooth-MPPI/smooth-MPPI.hpp>
