// TEST INFRASTRUCTURE — std_msgs/String (included, unused, by lesson4's hector_slam.h).
#pragma once
#include <string>
namespace std_msgs {
struct String { std::string data; };
}  // namespace std_msgs
