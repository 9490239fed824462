// TEST INFRASTRUCTURE — see tf_lesson4.h.
#pragma once
#include "tf/tf_lesson4.h"
