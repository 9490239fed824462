// TEST INFRASTRUCTURE — ros/console.h: the logging macros live in this stand-in's ros/ros.h.
#pragma once
#include "ros/ros.h"
