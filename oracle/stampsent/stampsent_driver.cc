// C-ABI driver of the C++ runtime's TimestampSentence (runtime/onnxruntime/src/util.cpp:569-637), compiled with util.cpp and
// encode_converter.cpp from the reference tree (Makefile beside this file).  util.cpp's parameter loader needs AlignedMalloc, which
// the checker never calls.
#include <stdlib.h>
#include <string.h>
#include <string>

namespace funasr {
void* AlignedMalloc(size_t alignment, size_t required_bytes) {
  void* p = nullptr;
  return posix_memalign(&p, alignment < sizeof(void*) ? sizeof(void*) : alignment, required_bytes) == 0 ? p : nullptr;
}
std::string TimestampSentence(std::string& text, std::string& str_time);
}  // namespace funasr

// the JSON string into out (NUL-terminated); returns its length, or -(length + 1) when cap is too small
extern "C" int stampsent_ref(const char* text, const char* stamp, char* out, int cap) {
  std::string t(text), s(stamp);
  const std::string r = funasr::TimestampSentence(t, s);
  if ((int)r.size() + 1 > cap) return -(int)r.size() - 1;
  memcpy(out, r.c_str(), r.size() + 1);
  return (int)r.size();
}
