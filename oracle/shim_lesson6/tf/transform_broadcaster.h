// TEST INFRASTRUCTURE — see tf_core.h.
#pragma once
#include "tf/tf_core.h"
