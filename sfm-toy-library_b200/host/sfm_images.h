// sfm_images.h -- SURVEY.md 8(f-3): the imread loop of SfM::setImagesDirectory (reference SfMToyLib/SfM.cpp:123-135) on the GPU.
//
//     for (auto& imageFilename : mImageFilenames) mImages.push_back(imread(imageFilename));
//
// becomes one call that reads every file and decodes all of them with sfmb200_decode_jpeg_batch: the same B,G,R bytes cv::imread
// returns (EXIF orientation applied), one upload and one download for the whole run.  Only JPEG files decode; there is no host
// fallback, so any other file (or a corrupt one) makes the call return false with the reason on std::cerr.
// The optional downscale of the loop (:127-129),
//
//     if (mDownscaleFactor != 1.0) resize(mImages.back(), mImages.back(), Size(), mDownscaleFactor, mDownscaleFactor);
//
// is the `downscale` argument: with a factor other than 1 every image is resized on the device in the same call
// (sfmb200_decode_jpeg_batch_scaled), byte-identical to cv::resize, and only the resized images are downloaded.
#pragma once
#include "sfmtoylib_b200.h"
#include <string>
#include <vector>

namespace sfmtoylib {

// Appends one CV_8UC3 image per file to `images`, in the order of `filenames`, resized by `downscale` unless it is 1.  false (and
// `images` unchanged) on any failure, including a factor cv::resize would refuse.
bool readImages(const std::vector<std::string>& filenames, std::vector<cv::Mat>& images, float downscale = 1.0f);

}  // namespace sfmtoylib
