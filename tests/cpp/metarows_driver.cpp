// tests/cpp/metarows_driver.cpp - TEST INFRASTRUCTURE for tests/golden/make_metarows_fixture.py.  Links against the unmodified
// reference (oracle/_ref/libkgref.a, built by oracle/Makefile.ref) and prints the SGF-metadata rows an SGF-metadata net is fed:
// SGFMetadata::fillMetadataRow (neuralnet/sgfmetadata.cpp) of the profile SGFMetadata::getProfile(NAME) gives, or of
// SGFMetadata::makeDummyWarmupProfile() for NAME "dummy_warmup", for a player to move and a board area.
//
//   metarows_driver NAME:PLAYER:AREA ...      PLAYER b or w
// prints one line per argument: NAME PLAYER AREA and the 192 floats of the row.
//   metarows_driver position RULES KOMI
// prints NNInputs::fillRowV7 (NHWC, no symmetry) of the empty 19x19 board, black to move, under Rules::parseRules(RULES) with that
// komi: "spatial" and the 22*361 floats, then "global" and the 19 floats - the position gtp's kata-raw-human-nn evaluates after
// clear_board.
#include "game/board.h"
#include "game/boardhistory.h"
#include "game/rules.h"
#include "neuralnet/nninputs.h"
#include "neuralnet/sgfmetadata.h"

#include <cstdio>
#include <string>
#include <vector>

int main(int argc, char** argv) {
  if(argc == 4 && std::string(argv[1]) == "position") {
    Board::initHash();
    Rules rules = Rules::parseRules(argv[2]);
    rules.komi = std::stof(argv[3]);
    Board board(19, 19);
    BoardHistory hist(board, P_BLACK, rules, 0, false);   // no stone is pass-alive on an empty board either way
    MiscNNInputParams params;
    std::vector<float> spatial(22 * 361), global(19);
    NNInputs::fillRowV7(board, hist, P_BLACK, params, 19, 19, true, spatial.data(), global.data());
    printf("spatial");
    for(float v : spatial) printf(" %.9g", v);
    printf("\nglobal");
    for(float v : global) printf(" %.9g", v);
    printf("\n");
    return 0;
  }
  for(int i = 1; i < argc; i++) {
    const std::string arg = argv[i];
    const size_t a = arg.find(':'), b = arg.rfind(':');
    if(a == std::string::npos || a == b) { fprintf(stderr, "bad argument %s\n", argv[i]); return 1; }
    const std::string name = arg.substr(0, a), pla = arg.substr(a + 1, b - a - 1);
    const int area = std::stoi(arg.substr(b + 1));
    const SGFMetadata meta = name == "dummy_warmup" ? SGFMetadata::makeDummyWarmupProfile() : SGFMetadata::getProfile(name);
    std::vector<float> row(SGFMetadata::METADATA_INPUT_NUM_CHANNELS);
    SGFMetadata::fillMetadataRow(&meta, row.data(), pla == "b" ? P_BLACK : P_WHITE, area);
    printf("%s %s %d", name.c_str(), pla.c_str(), area);
    for(float v : row) printf(" %.9g", v);
    printf("\n");
  }
  return 0;
}
