// The host's libstdc++ generator and distributions, as include/rrt.h uses them, for tests/test_rrt.py to compare the
// checker's restatement with.  Built with -Wall -Werror.
//   rrt_dist_pin mt   IN OUT       IN: uint32 seeds; OUT: 100000 outputs of std::mt19937(seed) per seed (uint32)
//   rrt_dist_pin int  IN OUT       IN: uint32 generator values fed through a URBG with mt19937's result_type, min
//   rrt_dist_pin real IN OUT A B   and max; OUT: (result, values used) int32 pairs of uniform_int_distribution<int>(0,
//                                  100), or of uniform_real_distribution<float>(A, B) with the result's float bits,
//                                  until the values run out
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <vector>

struct Crafted {  // a URBG that replays fixed values
  typedef std::mt19937::result_type result_type;
  static constexpr result_type min() { return std::mt19937::min(); }
  static constexpr result_type max() { return std::mt19937::max(); }
  const std::vector<uint32_t>* v;
  size_t pos;
  struct Dry {};
  result_type operator()() {
    if (pos >= v->size()) throw Dry();
    return (*v)[pos++];
  }
};

static std::vector<uint32_t> slurp(const char* path) {
  std::vector<uint32_t> v;
  FILE* f = std::fopen(path, "rb");
  if (!f) std::exit(2);
  uint32_t x;
  while (std::fread(&x, 4, 1, f) == 1) v.push_back(x);
  std::fclose(f);
  return v;
}

int main(int argc, char** argv) {
  if (argc < 4) return 2;
  const std::vector<uint32_t> in = slurp(argv[2]);
  std::vector<uint32_t> out;
  if (!std::strcmp(argv[1], "mt")) {
    for (uint32_t s : in) {
      std::mt19937 g(s);
      for (int i = 0; i < 100000; ++i) out.push_back((uint32_t)g());
    }
  } else {
    const bool real = !std::strcmp(argv[1], "real");
    if (real && argc != 6) return 2;
    std::uniform_int_distribution<int> di(0, 100);
    std::uniform_real_distribution<float> dr(real ? std::strtof(argv[4], 0) : 0.0f, real ? std::strtof(argv[5], 0) : 1.0f);
    Crafted g{&in, 0};
    try {
      for (;;) {
        const size_t p0 = g.pos;
        uint32_t r;
        if (real) {
          const float f = dr(g);
          std::memcpy(&r, &f, 4);
        } else {
          r = (uint32_t)di(g);
        }
        out.push_back(r);
        out.push_back((uint32_t)(g.pos - p0));
      }
    } catch (const Crafted::Dry&) {
    }
  }
  FILE* o = std::fopen(argv[3], "wb");
  if (!o) return 2;
  std::fwrite(out.data(), 4, out.size(), o);
  std::fclose(o);
  return 0;
}
