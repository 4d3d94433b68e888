// Stand-in for the C++ runtime's precomp.h when util.cpp / encode_converter.cpp are compiled alone for the TimestampSentence checker:
// the system headers they use, a LOG that discards its message, and the two headers whose functions the checker calls.
#pragma once
#include <assert.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <cstring>
#include <deque>
#include <fstream>
#include <iostream>
#include <iterator>
#include <list>
#include <map>
#include <memory>
#include <numeric>
#include <sstream>
#include <string>
#include <unordered_map>
#include <vector>

struct NullLog {
  template <typename T> NullLog& operator<<(const T&) { return *this; }
};
#define LOG(level) NullLog()

#include "util.h"
#include "encode_converter.h"
