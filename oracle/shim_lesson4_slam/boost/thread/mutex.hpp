// TEST INFRASTRUCTURE — boost::mutex for lesson4's HectorMapMutex.h: lesson6's Boost stand-in.
#pragma once
#include <boost/thread.hpp>
