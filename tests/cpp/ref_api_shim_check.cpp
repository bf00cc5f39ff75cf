// Executes the resampling<100>(), solve_DARE() and dlqr() shims of include/crb/reference_api.hpp and dumps what
// they return.  Linked against tests/cpp/mock_crb.c on a CPU-only machine (marshalling check) or against the
// real libcrb.so on an H100.  usage: ref_api_shim_check in.bin out.bin
//   in : seed, px[100][4] (Eigen 4xNP column-major), pw[100], A4[16] B4[4] Q4[16] R4, A5[25] B5[10] Q5[25] R5[4]
//   out: px[100][4], pw[100], draws[100], X4[16] K4[4], X5[25] K5[10]
#include <cstdio>
#include <crb/reference_api.hpp>

int main(int argc, char** argv) {
  if (argc != 3) return 2;
  std::vector<float> in(1 + 400 + 100 + 16 + 4 + 16 + 1 + 25 + 10 + 25 + 4);
  FILE* f = std::fopen(argv[1], "rb");
  if (!f || std::fread(in.data(), sizeof(float), in.size(), f) != in.size()) return 2;
  std::fclose(f);
  const float* p = in.data();
  const unsigned seed = (unsigned)*p++;
  crb::Mat<4, 100> px;
  crb::Mat<100, 1> pw;
  std::memcpy(px.data(), p, 400 * sizeof(float)); p += 400;
  std::memcpy(pw.data(), p, 100 * sizeof(float)); p += 100;
  crb::Matrix4f A4, Q4; crb::Vector4f B4;
  std::memcpy(A4.data(), p, 64); p += 16;
  std::memcpy(B4.data(), p, 16); p += 4;
  std::memcpy(Q4.data(), p, 64); p += 16;
  const float R4 = *p++;
  crb::Matrix5f A5, Q5; crb::Matrix52f B5; crb::Matrix2f R5;
  std::memcpy(A5.data(), p, 100); p += 25;
  std::memcpy(B5.data(), p, 40); p += 10;
  std::memcpy(Q5.data(), p, 100); p += 25;
  std::memcpy(R5.data(), p, 16); p += 4;
  std::vector<float> out;
  try {
    std::mt19937 gen(seed);
    std::uniform_real_distribution<> uni_d(1.0, 2.0);
    resampling<100>(px, pw, gen, uni_d);            // by value: gen / uni_d are not advanced (:122-123)
    out.insert(out.end(), px.data(), px.data() + 400);
    out.insert(out.end(), pw.data(), pw.data() + 100);
    for (int i = 0; i < 100; ++i) out.push_back((float)uni_d(gen));   // hence these ARE the draws it used
    crb::Matrix4f X4 = solve_DARE(A4, B4, Q4, R4);
    crb::RowVector4f K4 = dlqr(A4, B4, Q4, R4);
    out.insert(out.end(), X4.data(), X4.data() + 16);
    out.insert(out.end(), K4.data(), K4.data() + 4);
    crb::Matrix5f X5 = solve_DARE(A5, B5, Q5, R5);
    crb::Matrix25f K5 = dlqr(A5, B5, Q5, R5);
    out.insert(out.end(), X5.data(), X5.data() + 25);
    out.insert(out.end(), K5.data(), K5.data() + 10);
  } catch (const std::exception& e) {
    std::fprintf(stderr, "%s\n", e.what());
    return 3;
  }
  f = std::fopen(argv[2], "wb");
  std::fwrite(out.data(), sizeof(float), out.size(), f);
  std::fclose(f);
  return 0;
}
