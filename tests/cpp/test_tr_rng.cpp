// gtsam's initializeRandomly draw, for tests/test_translation_recovery_cpu.py: one process-wide std::mt19937(42) and
// Point3(randomVal(rng), randomVal(rng), randomVal(rng)) with std::uniform_real_distribution<double>(-1, 1), built by g++ so
// that the three arguments are evaluated as the Linux gtsam wheel's compiler evaluates them.  Reads n, prints n points.
#include <cstdio>
#include <random>

struct Point3 {
  double x, y, z;
  Point3(double x_, double y_, double z_) : x(x_), y(y_), z(z_) {}
};

static std::mt19937 kRandomNumberGenerator(42);

int main() {
  int n = 0;
  if (std::scanf("%d", &n) != 1) return 1;
  std::uniform_real_distribution<double> randomVal(-1, 1);
  for (int i = 0; i < n; ++i) {
    const Point3 p(randomVal(kRandomNumberGenerator), randomVal(kRandomNumberGenerator), randomVal(kRandomNumberGenerator));
    std::printf("%.17g %.17g %.17g\n", p.x, p.y, p.z);
  }
  return 0;
}
