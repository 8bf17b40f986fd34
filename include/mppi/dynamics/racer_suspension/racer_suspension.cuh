// Source-compatibility forwarder: the reference's include path, served by the mppi_b200 host layer.
#pragma once
#include <mppi_b200/dynamics/racer_suspension/racer_suspension.hpp>
