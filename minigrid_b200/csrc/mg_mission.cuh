// mg_mission.cuh — a BabyAI mission code (mg_common.cuh: MIS_*) turned back into the reference's words: Instr.surface and
// ObjDesc.surface (babyai/core/verifier.py:64-100, 261, 294, 331, 378-384, 457, 498). One function, mission_words, feeds
// the three outputs of mg_mission.cu (the text, DictObservationSpaceWrapper's word indices and FlatObsWrapper's one-hot
// characters); it is host + device code, so the CPU tests run the same function through g++.
#pragma once
#include "mg_common.cuh"

namespace mg {

// the words of every mission the codes can express; colours in COLOR_TO_IDX order, object words in MIS_TYPE_* order
enum : int { MW_GO, MW_TO, MW_PICK, MW_UP, MW_OPEN, MW_PUT, MW_NEXT, MW_COMMA, MW_THEN, MW_AFTER, MW_YOU, MW_A, MW_THE,
             MW_RED, MW_GREEN, MW_BLUE, MW_PURPLE, MW_YELLOW, MW_GREY,
             MW_OBJECT, MW_KEY, MW_BALL, MW_BOX, MW_DOOR,
             MW_IN, MW_FRONT, MW_OF, MW_BEHIND, MW_ON, MW_YOUR, MW_LEFT, MW_RIGHT, MW_COUNT };
// a mission has at most 10 words ("open the purple door , then open the yellow door"; the comma is a word of its own)
constexpr int MISSION_MAX_WORDS = 16;
constexpr int MISSION_TEXT_BYTES = 96;  // FlatObsWrapper's maxStrLen (wrappers.py:573)
constexpr int MISSION_CHAR_CODES = 28;  // FlatObsWrapper's numCharCodes: a-z, space, comma

MG_HD const char *mission_word_text(int w) {
  switch (w) {
    case MW_GO: return "go";        case MW_TO: return "to";          case MW_PICK: return "pick";    case MW_UP: return "up";
    case MW_OPEN: return "open";    case MW_PUT: return "put";        case MW_NEXT: return "next";    case MW_COMMA: return ",";
    case MW_THEN: return "then";    case MW_AFTER: return "after";    case MW_YOU: return "you";      case MW_A: return "a";
    case MW_THE: return "the";      case MW_RED: return "red";        case MW_GREEN: return "green";  case MW_BLUE: return "blue";
    case MW_PURPLE: return "purple"; case MW_YELLOW: return "yellow"; case MW_GREY: return "grey";    case MW_OBJECT: return "object";
    case MW_KEY: return "key";      case MW_BALL: return "ball";      case MW_BOX: return "box";      case MW_DOOR: return "door";
    case MW_IN: return "in";        case MW_FRONT: return "front";    case MW_OF: return "of";        case MW_BEHIND: return "behind";
    case MW_ON: return "on";        case MW_YOUR: return "your";      case MW_LEFT: return "left";    default: return "right";
  }
}

// index in DictObservationSpaceWrapper.get_minigrid_words() (wrappers.py:475-531), -1 for the words it does not have
MG_HD int mission_word_vocab(int w) {
  switch (w) {
    case MW_RED: return 0;     case MW_GREEN: return 1;   case MW_BLUE: return 2;   case MW_YELLOW: return 3;
    case MW_PURPLE: return 4;  case MW_GREY: return 5;    case MW_BOX: return 10;   case MW_KEY: return 11;
    case MW_BALL: return 12;   case MW_DOOR: return 13;   case MW_PICK: return 17;  case MW_PUT: return 21;
    case MW_OPEN: return 23;   case MW_GO: return 24;     case MW_UP: return 29;    case MW_THE: return 30;
    case MW_A: return 31;      case MW_COMMA: return 33;  case MW_THEN: return 36;  case MW_TO: return 37;
    case MW_OF: return 38;     case MW_YOU: return 43;    case MW_OBJECT: return 47;
    default: return -1;
  }
}

// ObjDesc.surface: article, colour, type or "object", then the location phrase
MG_HD int mission_desc_words(uint32_t d, int *w, int n) {
  const uint32_t type = d & 7u, color = (d >> 3) & 7u, loc = (d >> 6) & 7u;
  w[n++] = ((d >> 9) & 1u) ? MW_A : MW_THE;
  if (color) w[n++] = MW_RED + (int)color - 1;
  w[n++] = MW_OBJECT + (int)(type <= MIS_TYPE_DOOR ? type : 0u);
  if (loc == MIS_LOC_FRONT) { w[n++] = MW_IN; w[n++] = MW_FRONT; w[n++] = MW_OF; w[n++] = MW_YOU; }
  else if (loc == MIS_LOC_BEHIND) { w[n++] = MW_BEHIND; w[n++] = MW_YOU; }
  else if (loc == MIS_LOC_LEFT || loc == MIS_LOC_RIGHT) { w[n++] = MW_ON; w[n++] = MW_YOUR; w[n++] = loc == MIS_LOC_LEFT ? MW_LEFT : MW_RIGHT; }
  return n;
}

// Instr.surface of a mission code as words (at most MISSION_MAX_WORDS); 0 words for MIS_CONST and unknown forms
MG_HD int mission_words(uint32_t code, int *w) {
  const uint32_t form = code & 7u, a = (code >> 3) & 1023u, b = (code >> 13) & 1023u;
  int n = 0;
  switch (form) {
    case MIS_GOTO: w[n++] = MW_GO; w[n++] = MW_TO; return mission_desc_words(a, w, n);
    case MIS_PICKUP: w[n++] = MW_PICK; w[n++] = MW_UP; return mission_desc_words(a, w, n);
    case MIS_OPEN: w[n++] = MW_OPEN; return mission_desc_words(a, w, n);
    case MIS_PUTNEXT:
      w[n++] = MW_PUT; n = mission_desc_words(a, w, n);
      w[n++] = MW_NEXT; w[n++] = MW_TO;
      return mission_desc_words(b, w, n);
    case MIS_BEFORE:
      w[n++] = MW_OPEN; n = mission_desc_words(a, w, n);
      w[n++] = MW_COMMA; w[n++] = MW_THEN; w[n++] = MW_OPEN;
      return mission_desc_words(b, w, n);
    case MIS_AFTER:
      w[n++] = MW_OPEN; n = mission_desc_words(a, w, n);
      w[n++] = MW_AFTER; w[n++] = MW_YOU; w[n++] = MW_OPEN;
      return mission_desc_words(b, w, n);
    default: return 0;
  }
}

// the mission string, zero padded to MISSION_TEXT_BYTES: words joined by spaces, a comma written straight after the word
// before it (BeforeInstr's ", then "); returns its length
MG_HD int mission_text(uint32_t code, uint8_t *out) {
  int w[MISSION_MAX_WORDS];
  const int nw = mission_words(code, w);
  int len = 0;
  for (int i = 0; i < MISSION_TEXT_BYTES; ++i) out[i] = 0;
  for (int i = 0; i < nw; ++i) {
    if (i > 0 && w[i] != MW_COMMA) out[len++] = ' ';
    for (const char *c = mission_word_text(w[i]); *c; ++c) out[len++] = (uint8_t)*c;
  }
  return len;
}

// DictObservationSpaceWrapper's row (string_to_indices with offset 1, zero padded to max_words): a word outside the
// vocabulary (the reference raises "Unknown word") is written as -1, and a mission longer than the row is cut (the
// reference asserts len < max_words_in_mission)
MG_HD void mission_indices(uint32_t code, int max_words, long long *out) {
  int w[MISSION_MAX_WORDS];
  const int nw = mission_words(code, w);
  for (int i = 0; i < max_words; ++i) {
    long long v = 0;
    if (i < nw) { const int k = mission_word_vocab(w[i]); v = k < 0 ? -1 : k + 1; }
    out[i] = v;
  }
}

// FlatObsWrapper's character code (wrappers.py:607-617): a-z 0..25, space 26, comma 27
MG_HD int mission_char_code(uint8_t ch) { return ch == ' ' ? 26 : ch == ',' ? 27 : (int)ch - 'a'; }

}  // namespace mg
