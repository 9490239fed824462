// TEST INFRASTRUCTURE — geometry_msgs/TwistStamped's header: the node only uses geometry_msgs::Twist (messages.h).
#pragma once

#include "geometry_msgs/messages.h"
