// TEST INFRASTRUCTURE — Boost as lesson6's karto_slam.cc uses it, on top of the stand-in open_karto already compiles
// against (oracle/shim/boost/thread.hpp): boost::bind (and its global placeholder _1) as std::bind, boost::mutex with
// scoped_lock, and boost::thread, which runs its function to completion when it is constructed.  The node's only thread
// is the transform-publish loop, which returns at once because ros::ok() is false in the stand-in.
#pragma once

#include <functional>
#include <mutex>

#include "../../shim/boost/thread.hpp"

using std::placeholders::_1;

namespace boost {
using std::bind;
struct mutex : std::mutex {
  typedef std::unique_lock<std::mutex> scoped_lock;
};
struct thread {
  template <class F>
  explicit thread(F f) { f(); }
  void join() {}
};
}  // namespace boost
