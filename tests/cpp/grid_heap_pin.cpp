// Drives the host's std::priority_queue<Node*, vector<Node*>, cmp> with cmp = left->key > right->key, the queue of
// src/a_star.cpp and src/dijkstra.cpp, through a sequence of pushes and pops, and writes the popped entries'
// insertion ids.  tests/test_grid.py compares them with the checker's restated heap (oracle/crb_oracle_grid.c).
//   argv[1]: ops.bin: n records of (uint8 op, float key): op 1 pushes key with id = record index, op 0 pops
//   argv[2]: out.bin: the popped ids, int32
#include <cstdint>
#include <cstdio>
#include <queue>
#include <vector>

struct Node {
  float key;
  int32_t id;
};

int main(int argc, char** argv) {
  if (argc != 3) return 2;
  FILE* in = std::fopen(argv[1], "rb");
  if (!in) return 2;
  std::vector<Node> nodes;
  std::vector<uint8_t> ops;
  uint8_t op;
  float key;
  while (std::fread(&op, 1, 1, in) == 1 && std::fread(&key, sizeof(float), 1, in) == 1) {
    ops.push_back(op);
    nodes.push_back(Node{key, (int32_t)nodes.size()});
  }
  std::fclose(in);
  auto cmp = [](const Node* left, const Node* right) { return left->key > right->key; };
  std::priority_queue<Node*, std::vector<Node*>, decltype(cmp)> pq(cmp);
  std::vector<int32_t> popped;
  for (size_t i = 0; i < ops.size(); ++i) {
    if (ops[i]) {
      pq.push(&nodes[i]);
    } else {
      if (pq.empty()) return 3;
      popped.push_back(pq.top()->id);
      pq.pop();
    }
  }
  FILE* o = std::fopen(argv[2], "wb");
  if (!o) return 2;
  std::fwrite(popped.data(), sizeof(int32_t), popped.size(), o);
  std::fclose(o);
  return 0;
}
