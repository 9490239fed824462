// TEST INFRASTRUCTURE — boost::lexical_cast<std::string> of a number, as lesson4's hector_slam.cc names its map topics.
#pragma once

#include <sstream>
#include <string>

namespace boost {
template <class T, class S>
T lexical_cast(const S &s) {
  std::ostringstream o;
  o << s;
  return o.str();
}
}  // namespace boost
